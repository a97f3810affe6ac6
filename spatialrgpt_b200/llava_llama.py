"""``LlavaLlamaModel`` — the reference's VLM class (llava/model/language_model/llava_llama.py:48-213
+ llava/model/llava_arch.py:252-650) re-built over the sm_90a kernels, keeping its public surface:
``generate(input_ids, images=, depths=, masks=, attention_mask=, **generation_kwargs)``, ``forward``,
``prepare_inputs_labels_for_multimodal``, ``encode_images``, the ``get_*`` accessors, ``config``,
``tokenizer``, ``device`` / ``dtype``.  ``LlavaLlamaForCausalLM`` is an alias (the name the north
star and llava/model/builder.py:138 use; the reference never defines it)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, List, Optional, Sequence, Tuple, Union

import torch

from . import logits_processors, ops
from .config import LlavaConfig
from .constants import IGNORE_INDEX, IMAGE_TOKEN_INDEX
from .llama_decoder import GenerateProbe, LlamaDecoder, PrefillProbe, check_candidates, sampling_warpers, sequence_seeds
from .multimodal_encoder import VisionTower
from .multimodal_projector import MultimodalProjector
from .region_extractor import RegionExtractor
from .splice_plan import SRC_TOKENS, build_splice_plan, reusable_prefix
from .weights import ModelWeights


@dataclass
class CausalLMOutputWithPast:
    logits: torch.Tensor
    loss: Optional[torch.Tensor] = None
    past_key_values: Any = None
    hidden_states: Any = None
    attentions: Any = None


@dataclass
class ScoreOutput:
    """LlavaLlamaModel.score: sequence_logprobs fp32 [B, N] (the sum over each candidate's tokens), token_logprobs fp32 [B, N, L_max]
    (0 past a candidate's length) and lengths int64 [N]."""
    sequence_logprobs: torch.Tensor
    token_logprobs: torch.Tensor
    lengths: torch.Tensor


@dataclass
class GenerateDecoderOnlyOutput:
    """generate(return_dict_in_generate=True) of greedy and sampled decoding, with HF's field names.  sequences: the int64 [rows, L]
    generate() returns without the flag.  scores (output_scores=True): one fp32 [rows, V] tensor per step, the row the step's token was
    chosen from (the raw row when greedy, after the logits processors when they are on, after the temperature / top-k / top-p warpers
    when sampled).  logits (output_logits=True): what generate(output_logits=True) returns beside the ids, one fp32 [n_b, V] per row."""
    sequences: torch.Tensor
    scores: Optional[Tuple[torch.Tensor, ...]] = None
    logits: Any = None
    attentions: Any = None
    hidden_states: Any = None
    past_key_values: Any = None


@dataclass
class GenerateBeamDecoderOnlyOutput:
    """generate(num_beams > 1, return_dict_in_generate=True), with HF's field names.  With output_scores=True: sequences_scores fp32 [B]
    (each prompt's best hypothesis' score, its summed log-probabilities over length ** length_penalty), scores (one fp32 [B * num_beams,
    V] log_softmax per step, before the beam score is added) and beam_indices int64 [B, L] (the row of each token of the hypothesis,
    -1 past its end)."""
    sequences: torch.Tensor
    sequences_scores: Optional[torch.Tensor] = None
    scores: Optional[Tuple[torch.Tensor, ...]] = None
    logits: Any = None
    beam_indices: Optional[torch.Tensor] = None
    attentions: Any = None
    hidden_states: Any = None
    past_key_values: Any = None


def refuse_batch_invariant(num_beams: int = 1, processors=None, lookup_k: int = 0, prefix_cache: bool = False, n_ret: int = 1,
                           output_scores: bool = False, llm=None) -> None:
    """The generate() options batch_invariant=True does not serve: raises NotImplementedError before any GPU work."""
    if num_beams != 1:
        raise NotImplementedError("batch_invariant=True with beam search")
    if processors is not None:
        raise NotImplementedError("batch_invariant=True with logits processors (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_length)")
    if lookup_k:
        raise NotImplementedError("batch_invariant=True with prompt_lookup_num_tokens")
    if prefix_cache:
        raise NotImplementedError("batch_invariant=True with prefix_cache=True")
    if n_ret != 1:
        raise NotImplementedError("batch_invariant=True with num_return_sequences > 1")
    if output_scores:
        raise NotImplementedError("batch_invariant=True with output_scores")
    if llm is not None and getattr(llm, "fp8", False):
        raise NotImplementedError("batch_invariant=True with quantization='fp8' (the rows step has no FP8 form)")
    if llm is not None and not getattr(llm, "supports_batch_invariant", False):
        raise NotImplementedError("batch_invariant=True on the tensor-parallel decoder")


def refuse_guidance(num_beams: int = 1, processors=None, lookup_k: int = 0, prefix_cache: bool = False, n_ret: int = 1,
                    output_scores: bool = False, llm=None) -> None:
    """The generate() options classifier-free guidance (guidance_scale != 1) does not serve: raises NotImplementedError before any GPU
    work.  Guided decoding runs each prompt and its unconditional branch as two rows of the rows step (LlamaDecoder.generate_rows)."""
    if num_beams != 1:
        raise NotImplementedError("guidance_scale with beam search (HF never reorders the unconditional branch's cache with the beams)")
    if processors is not None:
        raise NotImplementedError("guidance_scale with logits processors (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_length): "
                                  "the rows step runs none")
    if lookup_k:
        raise NotImplementedError("guidance_scale with prompt_lookup_num_tokens (the verify pass has no unconditional row)")
    if prefix_cache:
        raise NotImplementedError("guidance_scale with prefix_cache=True (guided prompts are prefilled whole)")
    if n_ret != 1:
        raise NotImplementedError("guidance_scale with num_return_sequences > 1")
    if output_scores:
        raise NotImplementedError("guidance_scale with output_scores (the guided rows are not returned)")
    if llm is not None and getattr(llm, "fp8", False):
        raise NotImplementedError("guidance_scale with quantization='fp8' (the rows step has no FP8 form)")
    if llm is not None and not getattr(llm, "supports_batch_invariant", False):
        raise NotImplementedError("guidance_scale on the tensor-parallel decoder (the rows step is a single-GPU kernel sequence)")


def refuse_contrastive(top_k: int = 50, processors=None, lookup_k: int = 0, prefix_cache: bool = False, return_logits: bool = False,
                       guided: bool = False, batch_invariant: bool = False, llm=None) -> None:
    """The generate() options contrastive search (penalty_alpha > 0, top_k > 1, greedy, one beam) does not serve: raises
    NotImplementedError before any GPU work.  Contrastive search runs every prompt's top_k candidates as rows of the batched step
    (LlamaDecoder.generate_contrastive)."""
    if top_k > 64:
        raise NotImplementedError(f"contrastive search with top_k = {top_k} > 64 (the candidates of a prompt are ranked in one CTA)")
    if processors is not None:
        raise NotImplementedError("penalty_alpha with logits processors (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_length)")
    if lookup_k:
        raise NotImplementedError("penalty_alpha with prompt_lookup_num_tokens (the verify pass checks greedy choices)")
    if prefix_cache:
        raise NotImplementedError("penalty_alpha with prefix_cache=True (the context needs every prompt row's hidden state)")
    if return_logits:
        raise NotImplementedError("penalty_alpha with output_logits")
    if guided:
        raise NotImplementedError("penalty_alpha with guidance_scale != 1")
    if batch_invariant:
        raise NotImplementedError("penalty_alpha with batch_invariant=True (the candidates run in the batched step)")
    if llm is not None and not getattr(llm, "supports_contrastive", False):
        raise NotImplementedError("penalty_alpha on the tensor-parallel decoder")


def group_beam_args(num_beams: int, num_beam_groups, diversity_penalty, do_sample: bool) -> Tuple[int, float]:
    """generate()'s num_beam_groups / diversity_penalty as (G, lambda), raising ValueError where transformers 4.37.2 does
    (GenerationConfig.validate, BeamSearchScorer, HammingDiversityLogitsProcessor): num_beams not a multiple of G or G > num_beams,
    do_sample with G > 1, lambda <= 0 with G > 1, lambda > 0 without groups.  G = 1 and lambda = 0 are plain beam search."""
    G = 1 if num_beam_groups is None else int(num_beam_groups)
    lam = 0.0 if diversity_penalty is None else float(diversity_penalty)
    if G < 1 or G > num_beams or num_beams % G:
        raise ValueError(f"num_beams ({num_beams}) has to be divisible by num_beam_groups ({G}), and num_beam_groups at most num_beams")
    if G > 1 and do_sample:
        raise ValueError("diverse beam search (num_beam_groups > 1) needs do_sample=False")
    if G > 1 and not lam > 0.0:
        raise ValueError(f"diverse beam search (num_beam_groups > 1) needs diversity_penalty > 0, got {diversity_penalty}")
    if G == 1 and lam > 0.0:
        raise ValueError("diversity_penalty > 0 needs num_beam_groups > 1 (HF's HammingDiversityLogitsProcessor)")
    return G, lam


def refuse_group_beams(processors=None, return_logits: bool = False, output_scores: bool = False, generate_outputs: bool = False,
                       prefix_cache: bool = False, lookup_k: int = 0, guided: bool = False, batch_invariant: bool = False, n_ret: int = 1,
                       llm=None) -> None:
    """The generate() options diverse beam search (num_beam_groups > 1) does not serve: raises NotImplementedError before any GPU work.
    Its groups run as the beams of the batched beam step (LlamaDecoder.generate_beam_batch with num_beam_groups)."""
    if processors is not None:
        raise NotImplementedError("num_beam_groups with logits processors (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_length)")
    if return_logits or output_scores:
        raise NotImplementedError("num_beam_groups with output_logits / output_scores")
    if generate_outputs:
        raise NotImplementedError("num_beam_groups with output_hidden_states / output_attentions")
    if prefix_cache:
        raise NotImplementedError("num_beam_groups with prefix_cache=True")
    if lookup_k:
        raise NotImplementedError("num_beam_groups with prompt_lookup_num_tokens")
    if guided:
        raise NotImplementedError("num_beam_groups with guidance_scale != 1")
    if batch_invariant:
        raise NotImplementedError("num_beam_groups with batch_invariant=True")
    if n_ret != 1:
        raise NotImplementedError("num_beam_groups with num_return_sequences > 1")
    if llm is not None and (not hasattr(llm, "generate_beam_batch") or type(llm).__name__ == "TPLlamaDecoder"):
        raise NotImplementedError("num_beam_groups on the tensor-parallel decoder")


def refuse_generate_outputs(num_beams: int = 1, contrastive: bool = False, guided: bool = False, batch_invariant: bool = False, lookup_k: int = 0,
                            prefix_cache: bool = False, n_ret: int = 1, return_logits: bool = False, n_prompts: int = 1, llm=None) -> None:
    """The generate() options output_hidden_states / output_attentions (with return_dict_in_generate=True) do not serve: raises
    NotImplementedError before any GPU work.  They are recorded by the probed prefill and the probed batch-1 / batched decode steps."""
    what = "output_hidden_states / output_attentions"
    if num_beams != 1:
        raise NotImplementedError(f"{what} with beam search")
    if contrastive:
        raise NotImplementedError(f"{what} with penalty_alpha (contrastive search)")
    if guided:
        raise NotImplementedError(f"{what} with guidance_scale != 1")
    if batch_invariant:
        raise NotImplementedError(f"{what} with batch_invariant=True")
    if lookup_k:
        raise NotImplementedError(f"{what} with prompt_lookup_num_tokens")
    if prefix_cache:
        raise NotImplementedError(f"{what} with prefix_cache=True")
    if n_ret != 1:
        raise NotImplementedError(f"{what} with num_return_sequences > 1")
    if return_logits and n_prompts > 1:
        raise NotImplementedError(f"{what} with output_logits over a batch (that path decodes the prompts one after another)")
    if llm is not None and not getattr(llm, "supports_generate_outputs", False):
        raise NotImplementedError(f"{what} on the tensor-parallel decoder: no rank holds every attention head")


def generate_outputs_bytes(L: int, H: int, nh: int, B: int, T: int, N: int, hidden: bool, attentions: bool) -> int:
    """Bytes of generate()'s hidden states / attentions for B prompts padded to T rows and N new tokens: the prompt step's (forward()'s
    outputs), then the N - 1 decode steps' [N - 1, L + 1, B, H] and [N - 1, L, B, nh, T + N - 1] element-type tensors."""
    N1 = max(int(N), 1) - 1
    return (2 * ((L + 1) * B * T * H * hidden + L * B * nh * T * T * attentions)
            + N1 * (L + 1) * B * H * 2 * hidden + N1 * L * B * nh * (T + N1) * 2 * attentions)


def contrastive_alpha(penalty_alpha) -> float:
    """generate()'s penalty_alpha as a float, ValueError unless it is a finite number in [0, 1]."""
    try:
        a = float(penalty_alpha)
    except (TypeError, ValueError):
        raise ValueError(f"penalty_alpha must be a number in [0, 1], got {penalty_alpha!r}") from None
    if isinstance(penalty_alpha, bool) or not math.isfinite(a) or not 0.0 <= a <= 1.0:
        raise ValueError(f"penalty_alpha must be a finite number in [0, 1], got {penalty_alpha!r}")
    return a


def negative_prompt_rows(negative_prompt_ids, negative_prompt_attention_mask, n_prompts: int, vocab_size: int) -> List[torch.Tensor]:
    """generate()'s negative_prompt_ids [B, T] (and optional attention mask [B, T], padding on either side) -> the B unpadded id rows
    (host int64).  Raises ValueError on a shape that does not match the B prompts, a mask that is not one non-empty run of ones per row,
    or an id outside [0, vocab_size) (IMAGE_TOKEN_INDEX included: the unconditional branch sees no images)."""
    ids = torch.as_tensor(negative_prompt_ids).detach().to("cpu")
    if ids.dim() != 2 or ids.shape[0] != n_prompts or ids.shape[1] < 1 or ids.dtype.is_floating_point:
        raise ValueError(f"negative_prompt_ids must be integer ids [{n_prompts}, T >= 1] (one row per prompt), got {tuple(ids.shape)}")
    ids = ids.to(torch.int64)
    lo, hi = int(ids.min()), int(ids.max())
    if lo < 0 or hi >= vocab_size:
        raise ValueError(f"negative_prompt_ids holds the id {lo if lo < 0 else hi}, outside the vocabulary [0, {vocab_size}) (image "
                         f"placeholders such as IMAGE_TOKEN_INDEX = {IMAGE_TOKEN_INDEX} have no place in the unconditional branch)")
    if negative_prompt_attention_mask is None:
        return list(ids.unbind(0))
    am = torch.as_tensor(negative_prompt_attention_mask).detach().to("cpu").bool()
    if tuple(am.shape) != tuple(ids.shape):
        raise ValueError(f"negative_prompt_attention_mask {tuple(am.shape)} does not match negative_prompt_ids {tuple(ids.shape)}")
    rows = []
    for b in range(n_prompts):
        idx = torch.nonzero(am[b]).flatten()
        if idx.numel() == 0 or int(idx[-1]) - int(idx[0]) + 1 != idx.numel():
            raise ValueError("negative_prompt_attention_mask needs every row to be one non-empty run of ones")
        rows.append(ids[b, int(idx[0]):int(idx[-1]) + 1])
    return rows


def batch_invariant_groups(B: int, size: int):
    """The (first, end) prompt ranges generate(batch_invariant=True) decodes one after another: groups of `size`, the last one shorter."""
    return [(lo, min(lo + size, B)) for lo in range(0, B, size)]


def stopping_fn_of(stopping_criteria):
    """generate()'s stopping_criteria as the decoders take it: a function of one row's ids so far that holds when any criterion
    holds for them as a batch of one; None without criteria."""
    if not stopping_criteria:
        return None
    return lambda ids: any(bool(c(ids[None], None)) for c in stopping_criteria)


def compute_transition_scores(sequences: torch.Tensor, scores, beam_indices: Optional[torch.Tensor] = None, normalize_logits: bool = False,
                              vocab_size: Optional[int] = None) -> torch.Tensor:
    """HF's GenerationMixin.compute_transition_scores: the score of every generated token, fp32 [rows, steps] (beams: [B, L], 0 where
    beam_indices is -1).  ``scores`` = generate()'s per-step tuple of [rows, V]; ``normalize_logits`` log-softmaxes each row first;
    ``beam_indices`` picks the row of each step for beam search.  Post-processing of returned tensors, in torch."""
    V = scores[0].shape[-1] if vocab_size is None else int(vocab_size)
    if beam_indices is None:
        beam_indices = torch.arange(scores[0].shape[0], device=sequences.device).view(-1, 1).expand(-1, len(scores))
    sc = torch.stack(scores).reshape(len(scores), -1).transpose(0, 1)  # [rows * V, steps]
    if normalize_logits:
        sc = torch.nn.functional.log_softmax(sc.reshape(-1, V, sc.shape[-1]), dim=1).reshape(-1, sc.shape[-1])
    mask = beam_indices < 0
    max_len = int((1 - mask.long()).sum(-1).max())
    beam_indices = beam_indices.clone()[:, :max_len]
    mask = mask[:, :max_len]
    beam_indices[mask] = 0
    cut = sequences.shape[-1] - max_len
    indices = sequences[:, cut:] + beam_indices * V
    out = sc.gather(0, indices)
    out[mask] = 0
    return out


class LlavaLlamaModel:
    config_class = LlavaConfig
    main_input_name = "input_embeds"

    def __init__(self, config: LlavaConfig, weights: ModelWeights, tokenizer=None, image_processor=None,
                 max_seq_len: int = 4096, tensor_parallel=None):
        """``tensor_parallel`` = None, or (rank, world[, process_group]): the Llama DECODE step is sharded over `world` ranks
        (tensor_parallel.py, BASELINE config c5); encoders and the prompt prefill stay replicated."""
        # fail loudly when the CUDA extension or an H100 is missing: there is no CPU path
        from . import _lib
        self.config = config
        self.weights = weights
        if self.dtype not in (torch.bfloat16, torch.float16):
            raise _lib.SrgptError(f"weights are {self.dtype}: the kernels compute in torch.bfloat16 or torch.float16")
        with ops.elem_dtype(self.dtype):
            _lib.load()
            if not torch.cuda.is_available():
                raise _lib.SrgptError("spatialrgpt_b200 needs a CUDA device (sm_90a); no CPU fallback exists")
            _lib.device_info()
        self.tokenizer = tokenizer
        self._image_processor = image_processor
        self._max_seq_len = max_seq_len
        self._tensor_parallel = tensor_parallel
        self.training = False
        config.model_dtype = str(self.dtype)
        self._build_modules()

    @ops.in_own_dtype
    def _build_modules(self) -> None:
        config, weights, image_processor, max_seq_len, tensor_parallel = (self.config, self.weights, self._image_processor, self._max_seq_len,
                                                                          self._tensor_parallel)
        self.vision_tower = VisionTower(config, weights.vision, image_processor)
        self.mm_projector = MultimodalProjector(config, weights.projector)
        self.region_extractor = RegionExtractor(config, weights.region) if (config.enable_region and weights.region is not None) else None
        if tensor_parallel is not None and int(tensor_parallel[1]) > 1:
            from .tensor_parallel import TPLlamaDecoder
            self.llm = TPLlamaDecoder(config.llama, weights.llama, int(tensor_parallel[0]), int(tensor_parallel[1]),
                                      group=tensor_parallel[2] if len(tensor_parallel) > 2 else None, max_seq_len=max_seq_len)
        else:
            self.llm = LlamaDecoder(config.llama, weights.llama, max_seq_len=max_seq_len)
        # generate(prefix_cache=True): what the previous such request left for the next one to reuse (see _encode_prefix_cached)
        self._prefix_state = None
        self.last_prefix_reuse = None
        self.last_speculation = None  # generate(prompt_lookup_num_tokens=k): (verify passes, tokens drafted, tokens accepted)
        self._last_plan_rows = None

    # ---- accessors (llava_arch.py:252-278) -----------------------------------------------------------
    def get_llm(self):
        return self.llm

    def get_lm_head(self):
        return self.weights.llama.lm_head

    def get_vision_tower(self):
        return self.vision_tower

    def get_mm_projector(self):
        return self.mm_projector

    def get_region_extractor(self):
        return self.region_extractor

    def get_input_embeddings(self):
        return self.llm.embed_tokens

    @property
    def device(self):
        return self.weights.llama.embed.device

    @property
    def dtype(self):
        """torch.bfloat16 or torch.float16 - the dtype of the weights, which is also the compute dtype (the matching build of the
        kernels is selected around every public call, ops.elem_dtype)."""
        return self.weights.dtype

    def eval(self):
        return self

    def cuda(self, *a, **k):
        return self

    def to(self, *a, **k):
        dt = k.get("dtype", None)
        for x in a:
            if isinstance(x, torch.dtype):
                dt = x
        if dt is not None and dt != self.dtype:
            # nn.Module.to(dtype): cast the weights and rebuild what is derived from them (rope tables, KV cache, decode graphs).
            # The reference's eval does exactly this after an fp16 load: model.to(dtype=torch.bfloat16) (eval_spatial.py:221).
            if dt not in (torch.bfloat16, torch.float16):
                raise NotImplementedError(f"the sm_90a path computes in torch.bfloat16 or torch.float16, not {dt}")
            self.weights.to(dt)
            self.config.model_dtype = str(dt)
            self._build_modules()
        return self

    # ---- encoders ---------------------------------------------------------------------------------
    @ops.in_own_dtype
    def encode_images(self, images: torch.Tensor) -> torch.Tensor:
        """llava_arch.py:307-310 (tower -> projector, no regions)."""
        return self.mm_projector(self.vision_tower(images))

    def _start_host_copies(self, tensors):
        """Device tensors -> pinned host copies on a side stream (None entries pass through).  Returns (host tensors, event):
        the caller synchronises the event, not the compute stream."""
        out, any_dev = [], False
        side = getattr(self, "_side_stream", None)
        for t in tensors:
            if t is None or not t.is_cuda:
                out.append(None if t is None else t.detach())
                continue
            if side is None:
                side = self._side_stream = torch.cuda.Stream(device=self.device)
            if not any_dev:
                side.wait_stream(torch.cuda.current_stream())
                any_dev = True
            with torch.cuda.stream(side):
                h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                h.copy_(t.detach(), non_blocking=True)
            out.append(h)
        if not any_dev:
            return out, None
        ev = torch.cuda.Event()
        ev.record(side)
        return out, ev

    def _tokens_per_image(self) -> int:
        """Rows one <image> slot expands to: the projector's 2x2 down-sampling of the 27x27 refined map (regions on) or of the
        tower grid (base_projector.py:32-52)."""
        from .region_extractor import ADA_POOL
        side = ADA_POOL if (self.config.enable_region and self.region_extractor is not None) else self.config.vision.grid
        return self.mm_projector.tokens_out(side)

    @staticmethod
    def _stack_images(images):
        """A list of [3, R, R] / [n, 3, R, R] tensors, or [B, n, 3, R, R], or [N, 3, R, R] -> [N, 3, R, R]."""
        if isinstance(images, (list, tuple)):
            return torch.cat([im if im.dim() == 4 else im[None] for im in images], dim=0)
        return images.flatten(0, 1) if images.dim() == 5 else images

    def _encode_multimodal(self, images, masks, depths, keep: Optional[dict] = None):
        """llava_arch.py:387-411.  Returns (image_features [N,196,H], mask_embeds, depth_embeds).  ``keep`` (a dict) receives the
        encoder outputs a later request may reuse: image_features, hres (nested order) and depth_features."""
        cfg = self.config
        images = self._stack_images(images)
        if depths is not None:
            depths = self._stack_images(depths)
        N = images.shape[0]
        mask_embeds = depth_embeds = None
        use_depth = cfg.enable_region and cfg.enable_depth and depths is not None
        if cfg.enable_region and self.region_extractor is not None and masks is not None:
            # the mask -> pooling-weight kernels need only the masks: side stream, under the tower passes launched next
            g = cfg.vision.grid
            self.region_extractor.mask_pooling.precompute(masks, N, [(4 * g, ops.ORDER_NESTED)] + ([(g, ops.ORDER_ROWMAJOR)] if use_depth else []),
                                                          self.device)
        if use_depth and depths.shape == images.shape:
            # one tower pass over [images; depths] (same weights, llava_arch.py:398,404): twice the GEMM M
            both = self.vision_tower(torch.cat([images.to(self.device), depths.to(self.device).to(images.dtype)], dim=0))
            tower_features, depth_features = both[:N], both[N:]
        else:
            tower_features = self.vision_tower(images)
            depth_features = self.vision_tower(depths) if use_depth else None
        if cfg.enable_region and self.region_extractor is not None:
            hres, lres = self.region_extractor.feature_refinement_nested(tower_features.contiguous())
            mask_embeds, depth_embeds = self.region_extractor(hres, None if depth_features is None else depth_features.contiguous(),
                                                              masks, hres_order=ops.ORDER_NESTED)
        else:
            hres, lres = None, tower_features
        image_features = self.mm_projector(lres)
        if keep is not None:
            keep.update(image_features=image_features, hres=hres, depth_features=depth_features)
        return image_features, mask_embeds, depth_embeds

    def _encode_prefix_cached(self, images, masks, depths, state: dict):
        """The encoders of a generate(prefix_cache=True) request.  Compares the request's images, depth images and masks bitwise
        with the copies kept from the previous such request: ONE small device compare (srgpt_rows_equal) and ONE host sync at the
        start of the request, to learn the outcome.  When every image (and, with the depth branch, every depth image) is
        unchanged, both tower passes, the refinement and the projector are skipped and only the mask pooling and the region
        projectors run again (masks may have changed or grown, as in a multi-turn region chat).  Fills ``state`` with the
        per-image / per-region equality the prompt-prefix rule needs (splice_plan.reusable_prefix) and with what the next
        request may reuse."""
        cfg, dev = self.config, self.device
        images = self._stack_images(images).to(dev)
        N = images.shape[0]
        region_on = cfg.enable_region and self.region_extractor is not None
        use_depth = region_on and cfg.enable_depth and depths is not None
        depths = self._stack_images(depths).to(dev) if use_depth else None
        mask_list = (list(masks) if masks is not None else []) + [None] * N
        mask_list = [None if m is None else m.to(dev) for m in mask_list[:N]]
        prev = self._prefix_state if (self._prefix_state is not None and self._prefix_state.get("images") is not None) else None

        counts = [0 if m is None else int(m.shape[0]) for m in mask_list]
        offs = [sum(counts[:i]) for i in range(N + 1)]
        flags = torch.zeros(2 * N + offs[N], dtype=torch.int32, device=dev)

        def compare(a, b, lo):  # rows of a vs b -> flags[lo:lo + a.shape[0]] when shapes / dtypes allow a bitwise comparison
            if a is None or b is None or a.dtype != b.dtype or a.shape[1:] != b.shape[1:] or a.shape[0] == 0:
                return
            n = min(a.shape[0], b.shape[0])
            ops.rows_equal(a[:n].contiguous(), b[:n].contiguous(), flags[lo:lo + n])

        if prev is not None and prev["images"].shape[0] == N and (prev["depths"] is None) == (depths is None):
            compare(images, prev["images"], 0)
            if depths is not None:
                compare(depths, prev["depths"], N)
            prev_offs = prev["mask_offs"]
            for i in range(N):
                if i < len(prev["masks"]) and prev_offs[i] == offs[i]:
                    compare(mask_list[i], prev["masks"][i], 2 * N + offs[i])
        eq = flags.cpu().bool().tolist()  # the one host sync of a prefix-cached request
        image_equal = [eq[i] and (depths is None or eq[N + i]) for i in range(N)]
        mask_equal = [eq[2 * N + offs[i] + k] and image_equal[i] for i in range(N) for k in range(counts[i])]
        skip = prev is not None and N > 0 and all(image_equal)
        state.update(images=prev["images"] if skip else images.clone(), depths=prev["depths"] if skip else (None if depths is None else depths.clone()),
                     masks=[None if m is None else m.contiguous().clone() for m in mask_list], mask_offs=offs, image_equal=image_equal,
                     mask_equal=mask_equal, encoders_skipped=skip)
        if not skip:
            return self._encode_multimodal(images, masks, depths, keep=state)
        # the encoder outputs of the previous request are this request's
        state.update(image_features=prev["image_features"], hres=prev["hres"], depth_features=prev["depth_features"])
        mask_embeds = depth_embeds = None
        if region_on and masks is not None:
            mask_embeds, depth_embeds = self.region_extractor(state["hres"], state["depth_features"], mask_list, hres_order=ops.ORDER_NESTED)
        return state["image_features"], mask_embeds, depth_embeds

    # ---- embedding splice (llava_arch.py:333-650) -----------------------------------------------------
    @ops.in_own_dtype
    def prepare_inputs_labels_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels, images,
                                             masks=None, depths=None, _packed_only: bool = False, _prefix: Optional[dict] = None):
        if images is None or (input_ids is not None and input_ids.shape[1] == 1):
            return input_ids, position_ids, attention_mask, past_key_values, None, labels  # llava_arch.py:355-385
        cfg = self.config
        dev = self.device
        # The splice plan needs only host-side facts (token ids, images / regions per request).  Order of events: (1) the ids
        # (and masks / labels) start their device->host copy on a side stream, (2) the encoders are launched, (3) the host
        # builds the plan while the GPU runs the tower, (4) plan upload + one gather kernel.  The host never waits on the tower
        # and the GPU never waits on the Python loop below (it cost ~15 % of a 32-request batch when it came in between).
        host_copies, copy_done = self._start_host_copies([input_ids, attention_mask, labels])
        encoded = self._encode_multimodal(images, masks, depths) if _prefix is None else self._encode_prefix_cached(images, masks, depths, _prefix)
        if copy_done is not None:
            copy_done.synchronize()
        ids_cpu = host_copies[0].to(torch.int64)
        B, T = ids_cpu.shape
        am_cpu = torch.ones((B, T), dtype=torch.bool) if attention_mask is None else host_copies[1].bool()
        lab_cpu = torch.full((B, T), IGNORE_INDEX, dtype=torch.int64) if labels is None else host_copies[2].to(torch.int64)
        if isinstance(images, (list, tuple)):
            n_img = sum(im.shape[0] if im.dim() == 4 else 1 for im in images)
        else:
            n_img = images.shape[0] * images.shape[1] if images.dim() == 5 else images.shape[0]
        n_tok = self._tokens_per_image()
        region_on = cfg.enable_region and self.region_extractor is not None
        depth_on = region_on and cfg.enable_depth and depths is not None
        mask_list = (list(masks) if masks is not None else []) + [None] * n_img
        plan = build_splice_plan(ids_cpu, None if attention_mask is None else am_cpu, None if labels is None else lab_cpu, n_tok,
                                 [0 if m is None else int(m.shape[0]) for m in mask_list[:n_img]], [m is not None for m in mask_list[:n_img]],
                                 cfg.llm_mask_token_id, cfg.llm_depth_token_id, region_on, depth_on,
                                 getattr(cfg.llama, "tokenizer_model_max_length", None), vocab_size=self.weights.llama.embed.shape[0])
        for w in plan.warnings:
            print(w)
        lens, new_labels = plan.lens, plan.labels
        self._last_plan_rows = (plan.src_id, plan.src_row)
        if _prefix is not None:
            _prefix.update(src_id=plan.src_id, src_row=plan.src_row, n_tok=n_tok)
        sid_dev, srow_dev = plan.src_id.to(dev, non_blocking=True), plan.src_row.to(dev, non_blocking=True)

        # ---- ONE gather kernel builds the embeddings of the whole batch from the encoder outputs
        image_features, mask_embeds, depth_embeds = encoded
        if tuple(image_features.shape[:2]) != (n_img, n_tok):
            raise RuntimeError(f"splice plan expected {(n_img, n_tok)} image tokens, encoders produced {tuple(image_features.shape[:2])}")
        H = image_features.shape[2]

        def cat_rows(embeds):
            parts = [] if embeds is None else [e for e in embeds if e is not None]
            return torch.cat(parts, 0).contiguous() if parts else None

        mflat, dflat = cat_rows(mask_embeds), cat_rows(depth_embeds)
        img_flat = image_features.reshape(n_img * n_tok, H)
        packed = ops.splice_rows(self.weights.llama.embed, img_flat, mflat if mflat is not None else img_flat,
                                 dflat if dflat is not None else img_flat, sid_dev, srow_dev)
        self._last_packed = (packed, lens)
        self._last_seq_lens = lens
        if _packed_only:  # generate(): the unpadded rows are what the decoder consumes (no [B, max_len, H] copy)
            return None, None, attention_mask, past_key_values, None, None
        new_embeds = list(torch.split(packed, lens, 0))

        max_len = max(x.shape[0] for x in new_embeds)
        left = getattr(cfg.llama, "tokenizer_padding_side", "right") == "left"
        out = torch.zeros((B, max_len, H), dtype=self.dtype, device=dev)
        lab_out = torch.full((B, max_len), IGNORE_INDEX, dtype=torch.int64)
        am_out = torch.zeros((B, max_len), dtype=torch.bool)
        pos_out = torch.zeros((B, max_len), dtype=torch.int64)
        for b, (e, l) in enumerate(zip(new_embeds, new_labels)):
            n = e.shape[0]
            sl = slice(max_len - n, max_len) if left else slice(0, n)
            out[b, sl] = e
            lab_out[b, sl] = l
            am_out[b, sl] = True
            pos_out[b, sl] = torch.arange(n)
        ret_labels = None if labels is None else lab_out.to(dev)
        ret_am = None if attention_mask is None else am_out.to(device=dev, dtype=attention_mask.dtype)
        ret_pos = None if position_ids is None else pos_out.to(dev)
        self._last_seq_lens = [x.shape[0] for x in new_embeds]
        return None, ret_pos, ret_am, past_key_values, out, ret_labels

    # ---- forward: logits for every position (llava_llama.py:100-192) ----------------------------------
    @torch.no_grad()
    @ops.in_own_dtype
    def forward(self, input_ids=None, images=None, masks=None, depths=None, attention_mask=None, position_ids=None,
                past_key_values=None, seqlens_in_batch=None, inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, **kwargs):
        """Logits of every position (and the loss with ``labels``), as LlavaLlamaForCausalLM.forward.  ``output_hidden_states=True``:
        ``hidden_states`` is a tuple of L + 1 element-type [B, S, H] tensors, the embeddings, the residual stream after each layer but the
        last, and the final norm of the last (the rows lm_head reads).  ``output_attentions=True``: ``attentions`` is a tuple of L
        element-type [B, num_heads, S, S] tensors, each layer's causal softmax in fp32, cast.  Both are views of one allocation each, and
        are 0 at every padded position (query or key).  The logits and the loss are bit-identical with or without them."""
        if past_key_values is not None:
            raise NotImplementedError("external past_key_values are not supported; the KV cache is paged and internal")
        want_h, want_a = bool(output_hidden_states), bool(output_attentions)
        if want_h or want_a:
            if not getattr(self.llm, "supports_forward_outputs", False):
                raise NotImplementedError("output_hidden_states / output_attentions on the tensor-parallel decoder: no rank holds every attention head")
            if inputs_embeds is not None or images is None:  # the row count is known before any device work
                self._check_forward_outputs_fit(*(inputs_embeds.shape[:2] if inputs_embeds is not None else input_ids.shape), want_h, want_a)
        if inputs_embeds is None:
            if images is None:
                inputs_embeds = self.llm.embed_tokens(input_ids).view(*input_ids.shape, -1)
            else:
                (_, position_ids, attention_mask, _, inputs_embeds, labels) = self.prepare_inputs_labels_for_multimodal(
                    input_ids, position_ids, attention_mask, None, labels, images, masks, depths)
                if want_h or want_a:  # the spliced row count
                    self._check_forward_outputs_fit(*inputs_embeds.shape[:2], want_h, want_a)
        B, S, H = inputs_embeds.shape
        lens = [S] * B if attention_mask is None else attention_mask.bool().sum(-1).tolist()
        lens = [int(n) for n in lens]
        logits = torch.zeros((B, S, self.config.llama.vocab_size), dtype=torch.float32, device=self.device)
        valid = [slice(0, n) for n in lens]
        if attention_mask is not None:  # either padding side: the valid rows of a sequence are contiguous
            am = attention_mask.bool()
            for b in range(B):
                idx = torch.nonzero(am[b]).flatten()
                if idx.numel() != lens[b] or (lens[b] and int(idx[-1]) - int(idx[0]) + 1 != lens[b]):
                    raise NotImplementedError("attention masks with holes are not supported")
                valid[b] = slice(int(idx[0]), int(idx[0]) + lens[b]) if lens[b] else slice(0, 0)
        llm = self.llm
        for b in range(len(llm.cache.owned)):
            llm.cache.release(b)
        probe, hs, att = None, None, None
        if want_h or want_a:
            d = llm.dims
            L = d.num_hidden_layers
            if want_h:
                hs = torch.empty((L + 1, B, S, H), dtype=self.dtype, device=self.device)
                for b in range(B):  # the probed prefill writes the valid rows only
                    hs[:, b, :valid[b].start].zero_()
                    hs[:, b, valid[b].stop:].zero_()
            if want_a:  # every entry is written by the probability kernel, padding included
                att = torch.empty((L, B, d.num_attention_heads, S, S), dtype=self.dtype, device=self.device)
            probe = PrefillProbe(torch.tensor([v.start for v in valid], dtype=torch.int32).to(self.device), None if hs is None else hs[:L], att)
        if B == 1:
            hid = llm.prefill_hidden(inputs_embeds[0, valid[0]], 0, 0, **({} if probe is None else dict(probe=probe)))
        else:  # one packed pass over all rows of the batch
            llm.ensure_capacity(B, max(lens))
            llm.cache.reserve_many(lens)
            hid = llm.prefill_packed(torch.cat([inputs_embeds[b, valid[b]] for b in range(B)], 0), lens,
                                     **({} if probe is None else dict(probe=probe)))
        hn = None if hs is None else llm.final_norm(hid)  # hidden_states[L]: the very rows lm_head reads
        loss = None
        if labels is None:
            lg = llm.logits_all(hid, **({} if hn is None else dict(normed=hn)))
        else:  # the element-type rows the lm_head GEMM writes, plus one zero row: the logits this call returns at padding positions
            total = hid.shape[0]
            buf = llm._logits_buffer(total + 1)
            lg = llm.lm_head_rows(hid, out=buf[:total], **({} if hn is None else dict(normed=hn))).float()
            buf[total].zero_()
            loss = self._labels_loss(buf, labels, valid, lens, S)
        o = 0
        for b in range(B):
            logits[b, valid[b]] = lg[o:o + lens[b]]
            if hs is not None:
                hs[-1, b, valid[b]] = hn[o:o + lens[b]]
            o += lens[b]
        return CausalLMOutputWithPast(logits=logits, loss=loss, hidden_states=None if hs is None else tuple(hs.unbind(0)),
                                      attentions=None if att is None else tuple(att.unbind(0)))

    def _check_forward_outputs_fit(self, B: int, S: int, hidden: bool, attentions: bool) -> None:
        """RuntimeError naming the bytes forward()'s hidden states / attentions need when they exceed the free device memory."""
        d = self.llm.dims
        need = 2 * ((d.num_hidden_layers + 1) * B * S * d.hidden_size * hidden + d.num_hidden_layers * B * d.num_attention_heads * S * S * attentions)
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise RuntimeError(f"forward(output_hidden_states={hidden}, output_attentions={attentions}) over {B} x {S} rows needs {need} bytes "
                               f"({need / 2 ** 30:.1f} GiB) for its outputs; {free} bytes are free on {self.device}")

    @staticmethod
    def _labels_loss(elem_logits: torch.Tensor, labels: torch.Tensor, valid, lens, S: int) -> torch.Tensor:
        """LlamaForCausalLM.forward's loss (modeling_llama.py:1044-1058): CrossEntropyLoss over logits[:, :-1] against labels[:, 1:],
        IGNORE_INDEX skipped, mean over the batch.  ``elem_logits``: the packed element-type rows of the B sequences' valid positions and
        one zero row after them, which stands for every padding position.  One token_logprobs launch; the mean is taken on the device."""
        B = len(lens)
        lab = labels.detach().to("cpu", torch.int64)
        if tuple(lab.shape) != (B, S):
            raise ValueError(f"labels {tuple(lab.shape)} do not match the inputs [{B}, {S}]")
        rowmap = torch.full((B, S), sum(lens), dtype=torch.int32)  # the zero row
        o = 0
        for b in range(B):
            rowmap[b, valid[b]] = torch.arange(o, o + lens[b], dtype=torch.int32)
            o += lens[b]
        rows, targets = rowmap[:, :-1].reshape(-1), lab[:, 1:].reshape(-1)
        keep = targets != IGNORE_INDEX
        _, _, loss = ops.token_logprobs(elem_logits, rows[keep], targets[keep], loss=True)
        return loss

    __call__ = forward

    # ---- likelihood scoring of answer candidates ------------------------------------------------------------------------------------
    @torch.no_grad()
    @ops.in_own_dtype
    def score(self, input_ids: torch.Tensor, images=None, depths=None, masks=None, attention_mask=None, candidates=None) -> "ScoreOutput":
        """Rank answer candidates by likelihood: ``candidates`` is a list of N non-empty token-id lists shared by the B prompts.
        token_logprobs[b, c, j] = log p(cand_c[j] | prompt_b ++ cand_c[:j]), what forward() on the concatenation gives at those rows
        up to rounding, but each prompt is prefilled once and every candidate continues from its KV pages (LlamaDecoder.
        score_candidates).  Padding may be on either side of ``attention_mask``.  Raises ValueError on an empty candidate list or
        candidate, an id outside the vocabulary, or a prompt + candidate longer than the decoder's max_seq_len."""
        if not getattr(self.llm, "supports_scoring", False):
            raise NotImplementedError("likelihood scoring (score()) on the tensor-parallel decoder")
        cands = check_candidates(candidates, self.llm.dims.vocab_size)
        lengths = [len(c) for c in cands]
        if images is not None:
            self.prepare_inputs_labels_for_multimodal(input_ids, None, attention_mask, None, None, images, masks, depths, _packed_only=True)
            packed, lens = self._last_packed
            lens = [int(n) for n in lens]
        else:
            B, T = input_ids.shape
            rows = [slice(0, T)] * B
            if attention_mask is not None:
                am = attention_mask.bool().cpu()
                rows = []
                for b in range(B):
                    idx = torch.nonzero(am[b]).flatten()
                    if idx.numel() == 0 or int(idx[-1]) - int(idx[0]) + 1 != idx.numel():
                        raise ValueError("score() needs every prompt's attention mask to be one non-empty run of ones")
                    rows.append(slice(int(idx[0]), int(idx[-1]) + 1))
            lens = [r.stop - r.start for r in rows]
            if max(lens) + max(lengths) > self.llm.max_seq_len:
                raise ValueError(f"a prompt of {max(lens)} rows and a candidate of {max(lengths)} tokens exceed max_seq_len {self.llm.max_seq_len}")
            emb = self.llm.embed_tokens(input_ids)
            packed = torch.cat([emb[b * T + r.start:b * T + r.stop] for b, r in enumerate(rows)], 0)
        tok = self.llm.score_candidates(packed, lens, cands, self._score_row_budget(max(lengths)))
        return ScoreOutput(sequence_logprobs=tok.sum(-1), token_logprobs=tok, lengths=torch.tensor(lengths, dtype=torch.int64))

    def _score_row_budget(self, longest: int) -> int:
        """Rows of one scoring pass: a quarter of the free device memory over what a row costs (its element-type logits row and the
        chunked prefill's activations), between the longest candidate's rows and 8192."""
        d = self.llm.dims
        per_row = 2 * ((d.vocab_size + 7) // 8 * 8 + 3 * d.hidden_size + (2 * d.num_attention_heads + 2 * d.num_key_value_heads) * d.head_dim
                       + d.intermediate_size)
        free_b, _ = torch.cuda.mem_get_info(self.device)
        return int(max(longest - 1, 1, min(8192, free_b // 4 // per_row)))

    def _lookup_history(self, input_ids, attention_mask, multimodal: bool) -> torch.Tensor:
        """The prompt rows of a batch-1 request as prompt-lookup history: the token id of a text row, -1 (never matches) for a row
        taken from image features or region / depth embeddings (the splice plan's rows whose source is not the token table)."""
        if multimodal:
            sid, srow = self._last_plan_rows
            return torch.where(sid == SRC_TOKENS, srow, torch.full_like(srow, -1))
        ids = input_ids[0].cpu()
        if attention_mask is not None:
            ids = ids[attention_mask[0].cpu().bool()]
        return ids.to(torch.int32)

    # ---- generate (llava_llama.py:194-213) --------------------------------------------------------------
    @torch.no_grad()
    @ops.in_own_dtype
    def generate(self, input_ids: Optional[torch.Tensor] = None, images: Optional[torch.Tensor] = None,
                 depths: Optional[torch.Tensor] = None, masks: Optional[List[torch.Tensor]] = None,
                 attention_mask: Optional[torch.Tensor] = None, **generation_kwargs):
        do_sample = bool(generation_kwargs.pop("do_sample", False))
        temperature = generation_kwargs.pop("temperature", None)
        top_p = generation_kwargs.pop("top_p", None)
        top_k = generation_kwargs.pop("top_k", None)
        seed = generation_kwargs.pop("seed", None)
        num_beams = int(generation_kwargs.pop("num_beams", 1) or 1)
        max_new_tokens = generation_kwargs.pop("max_new_tokens", None)
        max_length = generation_kwargs.pop("max_length", None)
        generation_kwargs.pop("use_cache", None)
        stopping_criteria = generation_kwargs.pop("stopping_criteria", None)
        pad_token_id = generation_kwargs.pop("pad_token_id", None)
        eos_token_id = generation_kwargs.pop("eos_token_id", self.config.llama.eos_token_id)
        return_logits = bool(generation_kwargs.pop("output_logits", False))
        # return_dict_in_generate=True: an output object with HF's field names (GenerateDecoderOnlyOutput / GenerateBeamDecoderOnlyOutput);
        # with output_scores=True it carries the row each token was chosen from, written on the device by the decode step.  Without the
        # dict, output_scores is ignored, as HF ignores it.
        return_dict = bool(generation_kwargs.pop("return_dict_in_generate", False))
        output_scores = bool(generation_kwargs.pop("output_scores", False)) and return_dict
        # output_hidden_states / output_attentions (with the dict; ignored without it, as HF ignores them): HF's per-token tuples, entry 0
        # the prompt step (forward()'s outputs, bit for bit), entry t >= 1 decode step t, recorded on the device by the probed steps
        want_h = bool(generation_kwargs.pop("output_hidden_states", False)) and return_dict
        want_a = bool(generation_kwargs.pop("output_attentions", False)) and return_dict
        use_graph = bool(generation_kwargs.pop("use_cuda_graph", True))
        # prefix_cache=True (batch 1, opt-in): keep the previous such request's encoder outputs and the K/V of its prompt rows, and
        # prefill only the rows after the longest unchanged prefix (a follow-up turn of a conversation).  The new rows run through
        # short-M GEMMs and the paged attention kernel, so they differ from a full re-prefill by rounding; off, generate() is the
        # plain path.  model.last_prefix_reuse = (rows_reused, rows_prefilled, encoders_skipped) afterwards.
        prefix_cache = bool(generation_kwargs.pop("prefix_cache", False))
        # prompt_lookup_num_tokens=k (batch 1, greedy, opt-in; HF's prompt lookup decoding): draft up to k tokens by n-gram lookup
        # (sizes max_matching_ngram_size .. 1) and verify them in one pass over the weights.  The history searched is the prompt's text
        # ids (its image / mask / depth rows never match) plus the generated tokens; HF, given only inputs_embeds, searches the
        # generated tokens alone.  Either way the output does not depend on the drafts: ids and logits are bit-identical to
        # generate() without the option.  k above ops.SPEC_T_MAX - 1 is clamped to it (only the speed can tell).
        # model.last_speculation = (verify passes, tokens drafted, tokens accepted) afterwards.
        lookup_k = int(generation_kwargs.pop("prompt_lookup_num_tokens", 0) or 0)
        lookup_ngram = int(generation_kwargs.pop("max_matching_ngram_size", 2) or 2)
        # do_sample=True -> HF's TemperatureLogitsWarper + TopPLogitsWarper + multinomial, here one kernel per token
        # (eval_spatial.py:231-236 passes do_sample = temperature > 0, so temperature 0 stays greedy)
        # typical_p / epsilon_cutoff / eta_cutoff (HF's TypicalLogitsWarper, EpsilonLogitsWarper, EtaLogitsWarper after top-p, in that
        # order): applied by the same kernel when sampling; greedy decoding ignores them, as HF does.  typical_p <= 0 raises as HF's
        # warper does; typical_p >= 1 and cutoffs outside (0, 1) leave a warper off.
        warpers = {k: generation_kwargs.pop(k, None) for k in ("typical_p", "epsilon_cutoff", "eta_cutoff")}
        sampling = None
        if do_sample and temperature not in (0, 0.0):
            sampling = dict(temperature=1.0 if temperature is None else float(temperature), top_p=top_p, top_k=top_k, seed=seed, **warpers)
            sampling_warpers(sampling)  # the ValueError, before any device work
        # num_return_sequences=n (sampling): n answers per prompt, rows b * n .. b * n + n - 1 of the result (HF's repeat_interleave
        # order); each prompt is prefilled once and its n rows decode together in the batched sampled step
        n_ret = generation_kwargs.pop("num_return_sequences", None)
        n_ret = 1 if n_ret is None else int(n_ret)
        if n_ret < 1:
            raise ValueError(f"num_return_sequences must be >= 1, got {n_ret}")
        if n_ret > 1:
            if num_beams != 1:
                raise NotImplementedError("num_return_sequences > 1 with beam search (the n best hypotheses are not returned)")
            if sampling is None:
                raise ValueError("num_return_sequences > 1 needs do_sample=True with temperature > 0: greedy decoding has one answer per prompt")
            if prefix_cache:
                raise NotImplementedError("num_return_sequences > 1 with prefix_cache=True")
            if lookup_k:
                raise NotImplementedError("num_return_sequences > 1 with prompt_lookup_num_tokens")
            if return_logits:
                raise NotImplementedError("num_return_sequences > 1 with output_logits")
            if not getattr(type(self.llm), "supports_batch_sampling", False):
                raise NotImplementedError("num_return_sequences > 1 on the tensor-parallel decoder (it does not sample)")
        # batch_invariant=True (opt-in): row b of the result, ids and output_logits, equals bit for bit generate() of prompt b alone with the
        # same kwargs.  Each prompt runs the encoders and the prefill batch 1 runs; then up to ops.SPEC_T_MAX prompts decode together in
        # the rows step (LlamaDecoder.generate_rows), which streams each weight once and gives every row its one-token arithmetic.
        # ``seed`` may be a list of one seed per prompt; a scalar seed gives prompt b the seed sequence_seeds(seed, B)[b].
        batch_invariant = bool(generation_kwargs.pop("batch_invariant", False))
        # guidance_scale=g with negative_prompt_ids (opt-in; HF's UnbatchedClassifierFreeGuidanceLogitsProcessor): classifier-free guidance.
        # Each prompt's unconditional branch is the text model over its negative prompt (no images, masks or depth), continued by the
        # tokens chosen for the prompt; every token is chosen from g * (log_softmax(cond) - log_softmax(uncond)) + log_softmax(uncond).
        # The prompt and its branch decode as two rows of the rows step, so row b of the result equals a guided call of prompt b alone.
        # g = None or 1 is plain generate() (negative prompts ignored, as HF ignores them).
        guidance_scale = generation_kwargs.pop("guidance_scale", None)
        negative_prompt_ids = generation_kwargs.pop("negative_prompt_ids", None)
        negative_prompt_attention_mask = generation_kwargs.pop("negative_prompt_attention_mask", None)
        guided = guidance_scale is not None and float(guidance_scale) != 1.0
        # penalty_alpha=a with top_k=k (HF's contrastive search): when num_beams == 1, do_sample is false, a > 0 and k > 1 (top_k defaults
        # to 50, as HF's GenerationConfig), every token is chosen among the k most probable by (1 - a) * p - a * (the largest cosine of
        # the candidate's hidden state against the sequence's earlier ones).  Otherwise penalty_alpha is ignored, as HF ignores it.
        penalty_alpha = generation_kwargs.pop("penalty_alpha", None)
        contrastive_k = 50 if top_k is None else int(top_k)
        contrastive = (penalty_alpha is not None and contrastive_alpha(penalty_alpha) > 0.0 and contrastive_k > 1 and num_beams == 1
                       and not do_sample)
        length_penalty = float(generation_kwargs.pop("length_penalty", 1.0))
        early_stopping = bool(generation_kwargs.pop("early_stopping", False))
        # num_beam_groups=G with diversity_penalty=lambda (HF's group (diverse) beam search, transformers 4.37.2): the num_beams beams
        # form G groups chosen one after the other in every step, each token's log-prob lowered by lambda for every time an earlier
        # group of the prompt chose it in that step.  G = 1 with lambda = 0 is plain beam search.
        group_kw = {k: generation_kwargs.pop(k) for k in ("num_beam_groups", "diversity_penalty") if k in generation_kwargs}
        n_groups, diversity = group_beam_args(num_beams, group_kw.get("num_beam_groups"), group_kw.get("diversity_penalty"), do_sample) \
            if group_kw else (1, 0.0)
        # HF's logits processors (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_new_tokens / min_length), applied on the
        # device inside the decode step before the greedy choice or the sampling warpers (logits_processors.py, csrc/logits_process.cu).
        # The history is the generated tokens, as HF's given only inputs_embeds.  Neutral values leave generate() unchanged.
        proc_kw = {k: generation_kwargs.pop(k, None) for k in ("repetition_penalty", "no_repeat_ngram_size", "bad_words_ids", "min_new_tokens",
                                                              "min_length")}
        if num_beams != 1 and (sampling is not None or return_logits):
            raise NotImplementedError("beam search is implemented for do_sample=False without output_logits (the eval scripts' mode)")
        if generation_kwargs:
            raise TypeError(f"unsupported generation kwargs: {sorted(generation_kwargs)}")
        processors = logits_processors.parse(**proc_kw, eos_token_id=eos_token_id, vocab_size=getattr(self.config.llama, "vocab_size", None))
        if n_groups > 1:
            refuse_group_beams(processors=processors, return_logits=return_logits, output_scores=output_scores, generate_outputs=want_h or want_a,
                               prefix_cache=prefix_cache, lookup_k=lookup_k, guided=guided, batch_invariant=batch_invariant, n_ret=n_ret,
                               llm=self.llm)
        if processors is not None:
            if num_beams != 1:
                raise NotImplementedError("logits processors (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_length) with beam search")
            if lookup_k:
                raise NotImplementedError("logits processors with prompt_lookup_num_tokens (the verify pass would process every draft position)")
            if not getattr(self.llm, "supports_logits_processors", False):
                raise NotImplementedError("logits processors on the tensor-parallel decoder (its logits are vocabulary-parallel)")
        if lookup_k:
            if lookup_k < 0 or lookup_ngram < 1:
                raise ValueError("prompt_lookup_num_tokens and max_matching_ngram_size must be positive")
            if sampling is not None:
                raise NotImplementedError("prompt_lookup_num_tokens with do_sample=True (speculative sampling would change the random stream)")
            if num_beams != 1:
                raise NotImplementedError("prompt_lookup_num_tokens with beam search")
            if getattr(self.llm, "fp8", False):
                raise NotImplementedError("prompt_lookup_num_tokens with quantization='fp8' (the verify pass has no FP8 form)")
            if not getattr(self.llm, "supports_prompt_lookup", False):
                raise NotImplementedError("prompt_lookup_num_tokens on the tensor-parallel decoder")
        if num_beams != 1 and (not hasattr(self.llm, "generate_beam") or type(self.llm).__name__ == "TPLlamaDecoder"):
            raise NotImplementedError("beam search on the tensor-parallel decoder")
        if output_scores and not getattr(self.llm, "supports_output_scores", False):
            raise NotImplementedError("output_scores on the tensor-parallel decoder (its logits are vocabulary-parallel: no rank holds a whole row)")
        n_prompts = 1 if input_ids is None else int(input_ids.shape[0])
        if want_h or want_a:
            refuse_generate_outputs(num_beams=num_beams, contrastive=contrastive, guided=guided, batch_invariant=batch_invariant, lookup_k=lookup_k,
                                    prefix_cache=prefix_cache, n_ret=n_ret, return_logits=return_logits, n_prompts=n_prompts, llm=self.llm)
            if images is None:  # the prompt rows and the token budget are known before any device work
                B_, T_ = input_ids.shape
                lens_ = [T_] * B_ if attention_mask is None else [int(n) for n in attention_mask.sum(-1).tolist()]
                self._check_generate_outputs_fit(B_, T_, self._token_budget(max_new_tokens, max_length, lens_), want_h, want_a)
        if contrastive:
            refuse_contrastive(top_k=contrastive_k, processors=processors, lookup_k=lookup_k, prefix_cache=prefix_cache,
                               return_logits=return_logits, guided=guided, batch_invariant=batch_invariant, llm=self.llm)
        neg_rows = None
        if guided:
            refuse_guidance(num_beams=num_beams, processors=processors, lookup_k=lookup_k, prefix_cache=prefix_cache, n_ret=n_ret,
                            output_scores=output_scores, llm=self.llm)
            if negative_prompt_ids is None:
                raise ValueError("guidance_scale != 1 needs negative_prompt_ids: the prompt is given as embeddings, so HF's fallback (the "
                                 "last prompt id) does not exist here")
            neg_rows = negative_prompt_rows(negative_prompt_ids, negative_prompt_attention_mask, n_prompts, self.llm.dims.vocab_size)
        if isinstance(seed, (list, tuple)):
            if not batch_invariant and not guided:
                raise ValueError("a list of seeds needs batch_invariant=True")
            if len(seed) != n_prompts:
                raise ValueError(f"seed holds {len(seed)} seeds for {n_prompts} prompts")
        if guided:  # with or without batch_invariant=True: guided rows already decode batch-invariantly
            return self._generate_batch_invariant(input_ids, images, depths, masks, attention_mask, max_new_tokens, max_length, eos_token_id,
                                                  stopping_criteria, pad_token_id, use_graph, return_logits, return_dict, sampling, seed,
                                                  guidance=(float(guidance_scale), neg_rows))
        if batch_invariant:
            refuse_batch_invariant(num_beams=num_beams, processors=processors, lookup_k=lookup_k, prefix_cache=prefix_cache, n_ret=n_ret,
                                   output_scores=output_scores, llm=self.llm)
            if isinstance(seed, (list, tuple)) and sampling is not None:
                sampling["seed"] = int(seed[0]) if n_prompts == 1 else None
            if n_prompts > 1:
                return self._generate_batch_invariant(input_ids, images, depths, masks, attention_mask, max_new_tokens, max_length, eos_token_id,
                                                      stopping_criteria, pad_token_id, use_graph, return_logits, return_dict, sampling, seed)
        prefix = None
        if prefix_cache:
            if input_ids is None or input_ids.shape[0] != 1:
                raise NotImplementedError("prefix_cache=True serves batch-1 requests (no prefix sharing across a batch)")
            if num_beams != 1:
                raise NotImplementedError("prefix_cache=True with beam search")
            if not self.llm.supports_prefix_reuse:
                raise NotImplementedError("prefix_cache=True on the tensor-parallel decoder")
            prefix = {}

        packed = None
        if images is not None:
            self.prepare_inputs_labels_for_multimodal(input_ids, None, attention_mask, None, None, images, masks, depths, _packed_only=True,
                                                      _prefix=prefix)
            packed, lens = self._last_packed
            B = len(lens)
        else:
            inputs_embeds = self.llm.embed_tokens(input_ids).view(*input_ids.shape, -1)
            lens = [input_ids.shape[1]] * input_ids.shape[0] if attention_mask is None else attention_mask.sum(-1).tolist()
            B = inputs_embeds.shape[0]
            self._last_plan_rows = None
            if prefix is not None:  # text only: a row is its token id
                ids = input_ids[0].cpu() if attention_mask is None else input_ids[0].cpu()[attention_mask[0].cpu().bool()]
                prefix.update(src_id=torch.full((ids.numel(),), SRC_TOKENS, dtype=torch.int32), src_row=ids.to(torch.int32), n_tok=1,
                              image_equal=[], mask_equal=[], encoders_skipped=False)
        max_new_tokens = self._token_budget(max_new_tokens, max_length, lens)

        outs, all_logits = [], []
        left = getattr(self.config.llama, "tokenizer_padding_side", "right") == "left"
        gen_out, gp = None, None
        if want_h or want_a:  # the prompts' padded layout: generate()'s inputs_embeds, or the spliced rows padded as forward() pads them
            T_pad = int(inputs_embeds.shape[1]) if packed is None else max(int(n) for n in lens)
            if packed is not None:
                self._check_generate_outputs_fit(B, T_pad, int(max_new_tokens), want_h, want_a)
            gen_out, gp = self._generate_probe([int(n) for n in lens], T_pad, int(max_new_tokens), left, want_h, want_a)
        gp_kw = {} if gp is None else {"outputs": gp}
        extra = None  # the decoder's output_scores results
        sc_kw = {"output_scores": True} if output_scores else {}
        stop_fn = stopping_fn_of(stopping_criteria)
        lens = [int(n) for n in lens]
        processors = logits_processors.resolve_min_length(processors, max(lens))  # HF subtracts the (padded) inputs_embeds length
        proc = {} if processors is None else {"processors": processors}
        if lookup_k and B != 1:
            raise NotImplementedError("prompt_lookup_num_tokens serves batch-1 requests")
        if contrastive:  # any B: the prompts' unpadded rows, packed
            if packed is None:
                T = inputs_embeds.shape[1]
                packed = torch.cat([inputs_embeds[b, T - lens[b]:] if left else inputs_embeds[b, :lens[b]] for b in range(B)], 0)
            outs = self.llm.generate_contrastive(packed, lens, contrastive_k, contrastive_alpha(penalty_alpha), int(max_new_tokens),
                                                 eos_token_ids=eos_token_id, stopping_fn=stop_fn, use_graph=use_graph, **sc_kw)
            if output_scores:
                outs, extra = outs
        elif B == 1 and num_beams != 1 and n_groups == 1:
            n = lens[0]
            emb = packed if packed is not None else (inputs_embeds[0, inputs_embeds.shape[1] - n:] if left else inputs_embeds[0, :n])
            r = self.llm.generate_beam(emb, num_beams, int(max_new_tokens), eos_token_ids=eos_token_id, stopping_fn=stop_fn,
                                       length_penalty=length_penalty, early_stopping=early_stopping, use_graph=use_graph, **sc_kw)
            if output_scores:
                r, extra = r
            outs.append(r)
        elif B == 1 and n_ret == 1 and n_groups == 1:  # diverse beams of one prompt run the batched beam step below
            n = lens[0]
            emb = packed if packed is not None else (inputs_embeds[0, inputs_embeds.shape[1] - n:] if left else inputs_embeds[0, :n])
            reuse = 0
            if prefix is not None:
                prev = self._prefix_state
                self._prefix_state = None
                if prev is not None and prev["epoch"] == self.llm.prefix_epoch:  # no other request touched the cache since
                    reuse = reusable_prefix(prev["src_id"], prev["src_row"], prefix["src_id"], prefix["src_row"], prefix["n_tok"],
                                            prefix["image_equal"], prefix["mask_equal"], min(self.llm.prefix_rows, n - 1))
            spec = {}
            if lookup_k:
                spec = dict(lookup_ids=self._lookup_history(input_ids, attention_mask, packed is not None), lookup_k=lookup_k,
                            lookup_ngram=lookup_ngram)
            r = self.llm.generate_from_embeds(emb, int(max_new_tokens), eos_token_ids=eos_token_id, stopping_fn=stop_fn,
                                              use_graph=use_graph, return_logits=return_logits, sampling=sampling, reuse_rows=reuse, **spec,
                                              **proc, **sc_kw, **gp_kw)
            if output_scores:
                r, extra = r
            if lookup_k:
                self.last_speculation = tuple(self.llm.last_speculation)
            if prefix is not None:
                prefix["epoch"] = self.llm.prefix_epoch
                self._prefix_state = prefix
                self.last_prefix_reuse = (reuse, n - reuse, bool(prefix["encoders_skipped"]))
            if return_logits:
                r, lg = r
                all_logits.append(lg)
            outs.append(r)
        else:
            # batch > 1: one packed prefill over all prompts (llava_arch.py:549-611 pads, modeling_llama.py:540-562 unpads
            # again; here the rows were never padded), then batched decode (n_ret rows per prompt), or beam search with every prompt's
            # beams in one step
            if packed is None:
                T = inputs_embeds.shape[1]
                packed = torch.cat([inputs_embeds[b, T - lens[b]:] if left else inputs_embeds[b, :lens[b]] for b in range(B)], 0)
            if num_beams != 1:
                grp_kw = {} if n_groups == 1 else dict(num_beam_groups=n_groups, diversity_penalty=diversity, pad_token_id=pad_token_id)
                outs = self.llm.generate_beam_batch(packed, lens, num_beams, int(max_new_tokens), eos_token_ids=eos_token_id, stopping_fn=stop_fn,
                                                    length_penalty=length_penalty, early_stopping=early_stopping, use_graph=use_graph, **sc_kw,
                                                    **grp_kw)
                if output_scores:
                    outs, extra = outs
            else:
                r = self.llm.generate_batch(packed, lens, int(max_new_tokens), eos_token_ids=eos_token_id, stopping_fn=stop_fn,
                                            use_graph=use_graph, return_logits=return_logits, sampling=sampling, num_return_sequences=n_ret,
                                            **proc, **sc_kw, **gp_kw)
                if output_scores:
                    r, extra = r
                if return_logits:
                    outs, all_logits = r
                else:
                    outs = r
        res = self._generate_result(outs, pad_token_id, return_dict, all_logits if return_logits else None, extra, num_beams != 1)
        if gen_out is not None:
            res.hidden_states, res.attentions = self._generate_outputs(gen_out, max(o.numel() for o in outs))
        return res

    @staticmethod
    def _token_budget(max_new_tokens, max_length, lens) -> int:
        """generate()'s max_new_tokens: as given, else max_length less the longest prompt (at least 1), else HF's default max_length 20."""
        if max_new_tokens is not None:
            return max_new_tokens
        return 20 if max_length is None else max(int(max_length) - max(lens), 1)

    def _check_generate_outputs_fit(self, B: int, T: int, N: int, hidden: bool, attentions: bool) -> None:
        """RuntimeError naming the bytes generate()'s hidden states / attentions need (generate_outputs_bytes) when they exceed the free
        device memory."""
        d = self.llm.dims
        need = generate_outputs_bytes(d.num_hidden_layers, d.hidden_size, d.num_attention_heads, B, T, N, hidden, attentions)
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise RuntimeError(f"generate(output_hidden_states={hidden}, output_attentions={attentions}) over {B} x {T} prompt rows and {N} new "
                               f"tokens needs {need} bytes ({need / 2 ** 30:.1f} GiB) for its outputs; {free} bytes are free on {self.device}")

    def _generate_probe(self, lens: List[int], T: int, N: int, left: bool, hidden: bool, attentions: bool):
        """The tensors generate()'s hidden states / attentions live in, and the GenerateProbe that has the decoder record into them:
        the prompt step's [L + 1, B, T, H] / [L, B, nh, T, T] (forward()'s layout, 0 at padded rows) and the decode steps' [N - 1, L + 1,
        B, H] / [N - 1, L, B, nh, T + N - 1]; prompt b occupies rows / columns off_b .. off_b + n_b - 1, off_b = T - n_b when left."""
        d, dev, dt = self.llm.dims, self.device, self.dtype
        L, H, nh, B = d.num_hidden_layers, d.hidden_size, d.num_attention_heads, len(lens)
        offs = [T - n if left else 0 for n in lens]
        hs0 = hsd = att0 = attd = None
        if hidden:
            hs0 = torch.zeros((L + 1, B, T, H), dtype=dt, device=dev)
            hsd = torch.empty((N - 1, L + 1, B, H), dtype=dt, device=dev) if N > 1 else None
        if attentions:  # every entry of these is written by the probability kernels, padding included
            att0 = torch.empty((L, B, nh, T, T), dtype=dt, device=dev)
            attd = torch.empty((N - 1, L, B, nh, T + N - 1), dtype=dt, device=dev) if N > 1 else None
        off_dev = torch.tensor(offs, dtype=torch.int32).to(dev)
        steps = None
        if N > 1:
            steps = ops.StepProbe(off_dev, torch.tensor(lens, dtype=torch.int32).to(dev), T, hidden=hsd, attn=attd, step_offset=-1)
        gp = GenerateProbe(PrefillProbe(off_dev, None if hs0 is None else hs0[:L], att0), None if hs0 is None else hs0[L], offs, steps)
        return (hs0, att0, hsd, attd, T), gp

    @staticmethod
    def _generate_outputs(gen_out, n_max: int):
        """(hidden_states, attentions) of HF's generate(): one entry per token of the longest row, entry 0 the prompt step, entry t the
        decode step that read token t - 1 ([B, 1, H] per slot, [B, nh, 1, T + t] per layer), as views of the tensors _generate_probe made."""
        hs0, att0, hsd, attd, T = gen_out
        hs = att = None
        if hs0 is not None:
            hs = (tuple(hs0.unbind(0)),) + tuple(tuple(x[:, None] for x in hsd[t - 1].unbind(0)) for t in range(1, n_max))
        if att0 is not None:
            att = (tuple(att0.unbind(0)),) + tuple(tuple(x[:, :, None, :T + t] for x in attd[t - 1].unbind(0)) for t in range(1, n_max))
        return hs, att

    def _generate_batch_invariant(self, input_ids, images, depths, masks, attention_mask, max_new_tokens, max_length, eos_token_id, stopping_criteria,
                                  pad_token_id, use_graph: bool, return_logits: bool, return_dict: bool, sampling, seed, guidance=None):
        """generate(batch_invariant=True) over B > 1 prompts: every prompt's embeddings by the calls a batch-1 generate() of it makes (its
        unpadded ids; its images, depth images and masks), then groups of at most ops.SPEC_T_MAX prompts through generate_rows.
        ``guidance`` = (g, the B unpadded negative prompt id rows): classifier-free guidance for any B >= 1, in groups of at most
        ops.SPEC_T_MAX / 2 prompts (each with its unconditional row); a scalar seed of one prompt is its own seed, as in batch 1."""
        B = int(input_ids.shape[0])
        am = None if attention_mask is None else attention_mask.bool().cpu()
        ids_rows = [input_ids[b] if am is None else input_ids[b][am[b].to(input_ids.device)] for b in range(B)]
        if images is not None:
            counts = [int((r == IMAGE_TOKEN_INDEX).sum()) for r in ids_rows]
            all_images = self._stack_images(images)
            all_depths = None if depths is None else self._stack_images(depths)
            mask_list = (list(masks) if masks is not None else []) + [None] * all_images.shape[0]
            embeds, off = [], 0
            for b, ids in enumerate(ids_rows):
                k = counts[b]
                m = mask_list[off:off + k]
                m = None if all(x is None for x in m) else m  # a prompt without regions is called as batch 1 calls it: masks=None
                self.prepare_inputs_labels_for_multimodal(ids[None], None, None, None, None, all_images[off:off + k],
                                                          m, None if all_depths is None else all_depths[off:off + k], _packed_only=True)
                embeds.append(self._last_packed[0])
                off += k
        else:
            embeds = [self.llm.embed_tokens(ids) for ids in ids_rows]  # [n_b, H]
        lens = [int(e.shape[0]) for e in embeds]
        if max_new_tokens is not None:
            budgets = [int(max_new_tokens)] * B
        else:
            budgets = [20 if max_length is None else max(int(max_length) - n, 1) for n in lens]  # each row's own prompt length
        seeds = None
        if sampling is not None:
            if isinstance(seed, (list, tuple)):
                seeds = [int(s) for s in seed]
            elif guidance is not None and B == 1:
                seeds = [int(torch.initial_seed() if seed is None else seed)]
            else:
                seeds = sequence_seeds(torch.initial_seed() if seed is None else int(seed), B)
            sampling = dict(sampling, seed=None)
        stop_fn = stopping_fn_of(stopping_criteria)
        outs, all_logits = [], []
        guide, negs = {}, None
        if guidance is not None:
            negs = [self.llm.embed_tokens(r.to(self.device)) for r in guidance[1]]
            guide = dict(guidance_scale=guidance[0])
        for lo, hi in batch_invariant_groups(B, ops.SPEC_T_MAX // 2 if guidance is not None else ops.SPEC_T_MAX):
            if negs is not None:
                guide["negative_embeds"] = negs[lo:hi]
            r = self.llm.generate_rows(embeds[lo:hi], budgets[lo:hi], eos_token_ids=eos_token_id, stopping_fn=stop_fn, use_graph=use_graph,
                                       return_logits=return_logits, sampling=sampling, seeds=None if seeds is None else seeds[lo:hi], **guide)
            if return_logits:
                r, lg = r
                all_logits.extend(lg)
            outs.extend(r)
        return self._generate_result(outs, pad_token_id, return_dict, all_logits if return_logits else None)

    def _generate_result(self, outs: List[torch.Tensor], pad_token_id, return_dict: bool, logits=None, extra=None, beams: bool = False):
        """What generate() returns for the decoder's rows ``outs``: the ids [rows, longest] padded on the right with pad_token_id (the
        config's, else 0), with the fp32 ``logits`` of each row when output_logits, or as the return_dict_in_generate object, which
        also carries ``extra``, the decoder's output_scores results."""
        pad = pad_token_id if pad_token_id is not None else (self.config.llama.pad_token_id or 0)
        n_max = max(o.numel() for o in outs)
        seqs = torch.full((len(outs), n_max), int(pad), dtype=torch.int64, device=self.device)
        for b, o in enumerate(outs):
            seqs[b, : o.numel()] = o
        if not return_dict:
            return seqs if logits is None else (seqs, logits)
        scores = None if extra is None else tuple(extra["scores"].unbind(0))
        if not beams:
            return GenerateDecoderOnlyOutput(sequences=seqs, scores=scores, logits=logits)
        if extra is None:  # HF returns sequences_scores and beam_indices with output_scores only
            return GenerateBeamDecoderOnlyOutput(sequences=seqs)
        idx = torch.full(seqs.shape, -1, dtype=torch.int64)
        for b, bi in enumerate(extra["beam_indices"]):
            idx[b, : len(bi)] = torch.tensor(bi, dtype=torch.int64)
        return GenerateBeamDecoderOnlyOutput(sequences=seqs, sequences_scores=torch.tensor(extra["sequence_scores"], dtype=torch.float32,
                                                                                           device=self.device),
                                             scores=scores, beam_indices=idx.to(self.device))

    def compute_transition_scores(self, sequences: torch.Tensor, scores, beam_indices: Optional[torch.Tensor] = None,
                                  normalize_logits: bool = False) -> torch.Tensor:
        """HF's compute_transition_scores over generate(return_dict_in_generate=True, output_scores=True)'s sequences / scores /
        beam_indices: the score of every generated token (module-level compute_transition_scores)."""
        return compute_transition_scores(sequences, scores, beam_indices, normalize_logits, self.llm.dims.vocab_size)


LlavaLlamaForCausalLM = LlavaLlamaModel
