"""Region classification driver (COCO-80 / LVIS categories) over the sm_90a ``generate()`` path - the second caller of the hot
path in the reference, ``llava/eval/eval_region_cls.py`` (SURVEY.md §8f.3).  Same flags, same record format:

  annotation file (COCO format) -> one sample per non-crowd annotation (eval_region_cls.py:98-146)
  per sample: a square crop of the short image side around the box (49-72), the region as a segmentation mask or a box mask
  inside that crop (169-209), a randomly chosen "what is in <mask>" prompt + the dataset suffix (216-231), the conversation
  template, ``process_images`` / ``tokenizer_image_token`` (233-250), ``model.generate(..., max_new_tokens=64)`` (311-323) and
  one JSON line {question_id, text, gt_name, score, bbox, image_id, model_id, metadata} (333-346).

pycocotools is not a dependency here: polygon segmentations are rasterised with OpenCV (even-odd union of the polygons, like
``frPyObjects`` + ``decode`` summed over the parts), run-length ones with the decoder of eval_spatial.py.  The prompt choice uses a
seedable ``random.Random`` (the reference draws from the global generator)."""
from __future__ import annotations

import argparse
import copy
import json
import os
import random
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from .constants import DEFAULT_IMAGE_TOKEN, IMAGE_TOKEN_INDEX
from .conversation import conv_templates
from .eval_spatial import check_batch_size, clean_output, generate_invariant, get_chunk, pad_to_square, rle_decode, stop_string
from .mm_utils import _mask_processor, get_model_name_from_path, process_images, tokenizer_image_token

PROMPTS = [  # eval_region_cls.py:22-38 (data: the question pool of the benchmark)
    "Identify the object or feature present in the region denoted by <mask>.",
    "What category best describes the area represented by <mask>?",
    "Describe the content of the image section highlighted by <mask>.",
    "Can you specify the type of object or landscape within the bounds of <mask>?",
    "Which of the following categories best fits the region marked by <mask>? Provide your answer.",
    "What can you discern from the area indicated by <mask> in the image?",
    "Categorize the visual element within the area designated by <mask>.",
    "Give a brief description of the item or scene captured in the segment marked by <mask>.",
    "Which classification would you assign to the visual content found at <mask>?",
    "Determine and describe the primary subject located within <mask>.",
    "How would you label the section of the image encompassed by <mask>?",
    "Assess and classify the feature present within the confines of <mask>.",
    "If you were to tag the section indicated by <mask>, what tag would you use?",
    "What stands out to you in the region demarcated by <mask>? Please classify it.",
    "Evaluate the content of the image portion pinpointed by <mask> and provide its category.",
]


def get_crop_box(bboxes: List[List[float]], image_info: Dict[str, int]) -> List[int]:
    """eval_region_cls.py:49-72: a short_side x short_side window centred on the box, shifted back inside the image; the whole
    image when the box is larger than the short side.  (The reference compares the right / bottom edge with the SHORT side.)"""
    short = min(image_info["height"], image_info["width"])
    x1, y1, x2, y2 = bboxes[0]
    if y2 - y1 > short or x2 - x1 > short:
        return [0, 0, image_info["width"], image_info["height"]]
    cx, cy = int((x1 + x2) / 2), int((y1 + y2) / 2)
    xl, xr = cx - short // 2, cx + short // 2
    yt, yb = cy - short // 2, cy + short // 2
    if xl < 0:
        xl, xr = 0, short
    if xr > short:
        xl, xr = image_info["width"] - short, image_info["width"]
    if yt < 0:
        yt, yb = 0, short
    if yb > short:
        yt, yb = image_info["height"] - short, image_info["height"]
    return [xl, yt, xr, yb]


def generate_data_list(annotation_file: str) -> List[Dict[str, Any]]:
    """eval_region_cls.py:98-146: one entry per non-crowd annotation, boxes converted from xywh to xyxy, lower-cased category name."""
    with open(annotation_file) as f:
        coco = json.load(f)
    cid2name = {c["id"]: c["name"].lower() for c in coco.get("categories", [])}
    by_image: Dict[int, List[Dict[str, Any]]] = {}
    for ann in coco.get("annotations", []):
        by_image.setdefault(ann["image_id"], []).append(ann)
    out = []
    for img in sorted(coco.get("images", []), key=lambda i: i["id"]):
        parts = img["coco_url"].split("/")
        base = {"image": os.path.join("coco", parts[-2], parts[-1]), "image_info": {"height": img["height"], "width": img["width"]},
                "image_id": img["id"]}
        for ann in by_image.get(img["id"], []):
            if ann.get("iscrowd", 0) != 0:
                continue
            x, y, w, h = ann["bbox"]
            out.append(dict(copy.deepcopy(base), bbox=[[x, y, x + w, y + h]], segmentation=[copy.deepcopy(ann["segmentation"])],
                            category_name=cid2name[ann["category_id"]], score=1.0))
    return out


def segmentation_to_mask(segmentation, height: int, width: int) -> np.ndarray:
    """frPyObjects + decode + sum over the parts (eval_region_cls.py:186-189): polygons (list of flat [x0, y0, x1, y1, ...] lists)
    or an (un)compressed run-length dict."""
    if isinstance(segmentation, dict):
        return rle_decode(segmentation).astype(np.uint8)
    import cv2
    m = np.zeros((height, width), dtype=np.uint8)
    for poly in segmentation:
        part = np.zeros((height, width), dtype=np.uint8)
        pts = np.round(np.asarray(poly, dtype=np.float64).reshape(-1, 2)).astype(np.int32)
        cv2.fillPoly(part, [pts], 1)
        m += part  # overlapping parts add up, like np.sum(decode(...), axis=2)
    return m


def build_sample(line: Dict[str, Any], tokenizer, image_processor, model_config, conv_mode: str, dataset: str, prompt_type: str,
                 image_folder: str, rng: random.Random, open_image=None, return_conv: bool = False):
    """CustomDataset.__getitem__ (eval_region_cls.py:169-250) -> (input_ids [T], images [1, 3, R, R], masks [n, R, R]), and the
    conversation whose prompt the ids are when ``return_conv``."""
    from PIL import Image
    bboxes, info = line["bbox"], line["image_info"]
    assert len(bboxes) == 1, "one box per sample (eval_region_cls.py:177)"
    crop = get_crop_box(bboxes, info)
    pad = getattr(model_config, "image_aspect_ratio", None) == "pad"
    regions = []
    if prompt_type == "seg":
        for seg in line["segmentation"]:
            m = segmentation_to_mask(seg, info["height"], info["width"])[crop[1]:crop[3], crop[0]:crop[2]]
            regions.append(pad_to_square(m) if pad else m)
    else:
        for bbox in bboxes:
            m = np.zeros((info["height"], info["width"]), dtype=np.uint8)
            x1, y1, x2, y2 = map(int, bbox)
            m[y1:y2, x1:x2] = 1
            m = m[crop[1]:crop[3], crop[0]:crop[2]]
            regions.append(pad_to_square(m) if pad else m)
    mp = _mask_processor(image_processor)
    masks = torch.vstack([mp.preprocess(np.ascontiguousarray(m)[None, ...], return_tensors="pt")["pixel_values"][0] for m in regions]).float()
    question = rng.choice(PROMPTS)
    if len(bboxes) > 1:
        head, tail = question.split("<mask>")
        question = head + ",".join([" <mask>"] * (len(bboxes) - 1)) + " and <mask>" + tail
    question += (" Answer the question using a single word or phrase from COCO-80 categories." if dataset == "coco"
                 else " Answer the question using a single word or phrase from LVIS categories.")
    if getattr(model_config, "mm_use_im_start_end", False):
        raise ValueError("mm_use_im_start_end checkpoints are not supported by this benchmark (eval_region_cls.py:226-227)")
    conv = conv_templates[conv_mode].copy()
    conv.append_message(conv.roles[0], DEFAULT_IMAGE_TOKEN + "\n" + question)
    conv.append_message(conv.roles[1], None)
    image = (open_image or (lambda p: Image.open(p)))(os.path.join(image_folder, line["image"])).convert("RGB").crop(tuple(crop))
    images = process_images([image], image_processor, model_config)
    input_ids = tokenizer_image_token(conv.get_prompt(), tokenizer, IMAGE_TOKEN_INDEX, return_tensors="pt")
    return (input_ids, images, masks, conv) if return_conv else (input_ids, images, masks)


def category_names(annotation_file: str) -> List[str]:
    """The annotation file's category names, lower-cased as the records' gt_name, in the file's order."""
    with open(annotation_file) as f:
        return [c["name"].lower() for c in json.load(f).get("categories", [])]


def candidate_ids(conv, names: List[str], tokenizer, prompt_ids) -> List[List[int]]:
    """Each name as the template renders a final assistant turn (the conversation's open last turn answered with it), tokenised like
    the prompt: the ids after the prompt's, so each answer carries the template's own end-of-turn separator and a name that is a
    prefix of another is not favoured.  Raises ValueError when the prompt's ids are not a prefix of the answered prompt's."""
    prompt = [int(t) for t in prompt_ids.tolist()]
    out = []
    for name in names:
        c = conv.copy()
        c.messages[-1][1] = name
        full = tokenizer_image_token(c.get_prompt(), tokenizer, IMAGE_TOKEN_INDEX)
        if full[:len(prompt)] != prompt or len(full) == len(prompt):
            raise ValueError(f"the prompt's tokens are not a prefix of the tokens of the prompt answered with {name!r}")
        out.append(full[len(prompt):])
    return out


def eval_model(args, loader=None, seed: Optional[int] = None) -> int:
    """eval_region_cls.py:277-349.  ``loader`` defaults to ``load_pretrained_model``."""
    batch_size = int(getattr(args, "batch_size", 1) or 1)
    check_batch_size(batch_size, **{"--num_beams > 1": args.num_beams > 1, "--score-categories": getattr(args, "score_categories", False)})
    if loader is None:
        from .builder import load_pretrained_model as loader
    model_path = os.path.expanduser(args.model_path)
    model_name = get_model_name_from_path(model_path)
    quant = {"quantization": args.quantization} if getattr(args, "quantization", None) else {}
    if getattr(args, "nf4_planes_only", False):
        if getattr(args, "quantization", None) != "nf4":
            raise ValueError("--nf4-planes-only needs --quantization nf4")
        quant["nf4_dequantized_copy"] = False
    tokenizer, model, image_processor, _ = loader(model_path, model_name, getattr(args, "model_base", None), **quant)
    data = get_chunk(generate_data_list(args.annotation_file), args.num_chunks, args.chunk_idx)
    answers_file = os.path.expanduser(args.answers_file)
    os.makedirs(os.path.dirname(answers_file) or ".", exist_ok=True)
    rng = random.Random(seed)
    stop = stop_string(args.conv_mode)
    dev = model.device
    # --score-categories: rank the annotation file's category names by likelihood (model.score) instead of generating an answer
    names = category_names(args.annotation_file) if getattr(args, "score_categories", False) else None
    tails = {}  # prompt text -> the names' candidate ids
    n = 0
    gen_kw = dict(do_sample=args.temperature > 0, temperature=args.temperature, top_p=args.top_p, num_beams=args.num_beams, max_new_tokens=64,
                  use_cache=True)

    def record(line, text):
        return {"question_id": line["image"], "text": text, "gt_name": line["category_name"], "score": line["score"], "bbox": line["bbox"],
                "image_id": line["image_id"], "model_id": model_name, "metadata": {}}

    with open(answers_file, "w") as out:
        if batch_size > 1:
            # --batch-size N: N consecutive samples per generate(batch_invariant=True) call (the prompts drawn in the same order)
            for g in range(0, len(data), batch_size):
                lines = data[g:g + batch_size]
                samples = [build_sample(line, tokenizer, image_processor, model.config, args.conv_mode, args.dataset, args.prompt_type,
                                        args.image_folder, rng) for line in lines]
                seed = {"seed": [torch.initial_seed()] * len(lines)} if args.temperature > 0 else {}  # batch 1 draws with the default seed
                outs = generate_invariant(model, [ids.unsqueeze(0) for ids, _, _ in samples], torch.cat([im for _, im, _ in samples]).to(dev, dtype=model.dtype),
                                          None, [m.to(dev, dtype=model.dtype) for _, _, m in samples], **gen_kw, **seed)
                for line, output_ids in zip(lines, outs):
                    out.write(json.dumps(record(line, clean_output(tokenizer.batch_decode(output_ids, skip_special_tokens=True)[0], stop))) + "\n")
                    n += 1
                out.flush()
            return n
        for line in data:
            input_ids, images, masks, conv = build_sample(line, tokenizer, image_processor, model.config, args.conv_mode, args.dataset,
                                                          args.prompt_type, args.image_folder, rng, return_conv=True)
            # fp16 end to end, as the reference runs this script (builder.py:62 load, inputs cast at 316-317)
            if names is not None:
                key = conv.get_prompt()
                if key not in tails:
                    tails[key] = candidate_ids(conv, names, tokenizer, input_ids)
                res = model.score(input_ids.unsqueeze(0).to(dev), images=images.to(dev, dtype=model.dtype),
                                  masks=[masks.to(dev, dtype=model.dtype)], candidates=tails[key])
                text = names[int(res.sequence_logprobs[0].argmax())]
            else:
                output_ids = model.generate(input_ids.unsqueeze(0).to(dev), images=images.to(dev, dtype=model.dtype),
                                            masks=[masks.to(dev, dtype=model.dtype)], do_sample=args.temperature > 0,
                                            temperature=args.temperature, top_p=args.top_p, num_beams=args.num_beams, max_new_tokens=64,
                                            use_cache=True, pad_token_id=getattr(tokenizer, "pad_token_id", None))
                text = clean_output(tokenizer.batch_decode(output_ids, skip_special_tokens=True)[0], stop)
            out.write(json.dumps({"question_id": line["image"], "text": text, "gt_name": line["category_name"], "score": line["score"],
                                  "bbox": line["bbox"], "image_id": line["image_id"], "model_id": model_name, "metadata": {}}) + "\n")
            out.flush()
            n += 1
    return n


def build_arg_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="COCO / LVIS region classification over the sm_90a generate() path (flags of llava/eval/eval_region_cls.py)")
    p.add_argument("--model-path", type=str, required=True)
    p.add_argument("--model-base", type=str, default=None)
    p.add_argument("--image-folder", type=str, default="")
    p.add_argument("--annotation-file", type=str, default="")
    p.add_argument("--answers-file", type=str, default="answer.jsonl")
    p.add_argument("--conv-mode", type=str, default="llava_v1")
    p.add_argument("--num-chunks", type=int, default=1)
    p.add_argument("--chunk-idx", type=int, default=0)
    p.add_argument("--temperature", type=float, default=0.2)
    p.add_argument("--top_p", type=float, default=None)
    p.add_argument("--num_beams", type=int, default=1)
    p.add_argument("--dataset", type=str, default="lvis")
    p.add_argument("--prompt_type", type=str, default="seg")
    p.add_argument("--seed", type=int, default=None, help="seed of the prompt choice (the reference draws unseeded)")
    p.add_argument("--quantization", choices=["nf4", "fp8"], default=None,
                   help="quantization of the LLM's layer matrices: NF4 weight-only, or FP8 (E4M3) weights and activations")
    p.add_argument("--nf4-planes-only", action="store_true",
                   help="with --quantization nf4: keep only the 4-bit planes of the layer matrices, no dequantized copy (same answers)")
    p.add_argument("--score-categories", action="store_true",
                   help="answer with the category name of the highest likelihood under the prompt (model.score) instead of generating")
    p.add_argument("--batch-size", type=int, default=1,
                   help="answer this many consecutive samples in one generate(batch_invariant=True) call (same answers file)")
    return p


if __name__ == "__main__":
    _a = build_arg_parser().parse_args()
    print(f"wrote {eval_model(_a, seed=_a.seed)} answers")
