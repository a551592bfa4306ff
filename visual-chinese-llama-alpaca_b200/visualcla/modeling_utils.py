"""Chat / loader layer of the drop-in package (API boundary of SURVEY.md section 8b).

Mirrors the call signatures of ref: models/visualcla/modeling_utils.py --
`get_model_and_tokenizer_and_processor` (:83-141), `chat` (:143-178), `chat_in_stream` (:180-247),
`hijack_samplers` (:395-400), `DEFAULT_GENERATION_CONFIG` (:36-47) -- so that scripts/inference/*.py run
unchanged, while the model underneath is the H100-native engine.
"""
from __future__ import annotations

import gc
import logging
import os
import queue
import threading
from copy import deepcopy
from typing import List, Optional, Union

import torch
from transformers import GenerationConfig
from transformers.generation.logits_process import LogitsProcessor

from .configuration_visualcla import VisualCLAConfig
from .modeling_visualcla import VisualCLAModel

logger = logging.getLogger(__name__)

# The Alpaca-style multimodal prompt the checkpoints were trained with (ref: modeling_utils.py:28-34).
PROMPT_TEMPLATE_MULTIMODAL = (
    "Below is an instruction that describes a task. "
    "Write a response that appropriately completes the request.\n\n"
)
prompt_sep_before = "### "
prompt_sep_after = "\n\n"

DEFAULT_GENERATION_CONFIG = GenerationConfig(
    max_new_tokens=512, min_length=0, do_sample=True, top_p=0.9, top_k=40, num_beams=1, temperature=0.5,
    num_return_sequences=1, no_repeat_ngram_size=15, repetition_penalty=1.1,
)


def _turn(kind: str, body: str) -> str:
    if kind == "instruction":
        return f"{prompt_sep_before}Instruction: \n{body}{prompt_sep_after}"
    return f"{prompt_sep_before}Response:{body}{prompt_sep_after}"


def build_prompt(history: List[dict], text: str, image_block: str) -> str:
    """Conversation -> prompt string.  Only the first instruction of a conversation carries the image block
    (ref: modeling_utils.py:49-80): with an empty history that is the current turn, otherwise the history entry
    flagged `first_instruction`."""
    parts = [PROMPT_TEMPLATE_MULTIMODAL]
    for h in history:
        if h["type"] == "instruction":
            body = (image_block + "\n" + h["value"]) if "first_instruction" in h else h["value"]
            parts.append(_turn("instruction", body))
        elif h["type"] == "response":
            parts.append(_turn("response", h["value"]))
        else:
            raise ValueError(f"Except 'type' are 'instruction' and 'response', but get '{h['type']}'.")
    cur = (image_block + "\n" + text) if len(history) == 0 else text
    parts.append(f"{prompt_sep_before}Instruction: \n{cur}{prompt_sep_after}{prompt_sep_before}Response:")
    return "".join(parts)


def encoding_text(history, text, num_patch, tokenizer):
    image_block = tokenizer.img_start_token + num_patch * tokenizer.img_token + tokenizer.img_end_token
    prompt = tokenizer.bos_token + build_prompt(history, text, image_block)
    return tokenizer(prompt, return_tensors="pt", add_special_tokens=False)


def _attach_image_tokens(tokenizer):
    # ref: modeling_utils.py:94-102 -- ids are always resolved through the tokenizer
    tokenizer.pad_token = "<pad>"
    tokenizer.img_start_token = "<img>"
    tokenizer.img_end_token = "</img>"
    tokenizer.img_token = "<img_token>"
    tokenizer.img_start_token_id = tokenizer.convert_tokens_to_ids(tokenizer.img_start_token)
    tokenizer.img_end_token_id = tokenizer.convert_tokens_to_ids(tokenizer.img_end_token)
    tokenizer.img_token_id = tokenizer.convert_tokens_to_ids(tokenizer.img_token)
    return tokenizer


def get_model_and_tokenizer_and_processor(visualcla_model=None, text_model=None, vision_model=None, lora_model=None,
                                          torch_dtype=torch.float16, default_device=None, device_map=None,
                                          load_in_8bit=False, reuse_kv_cache=False, **engine_kwargs):
    """Same signature and return triple as the reference loader (:83-141).  `engine_kwargs` (max_batch, max_seq,
    max_prefill_tokens) size the device arenas of the H100 engine; reuse_kv_cache=True makes chat() / chat_in_stream() keep
    the KV cache between turns (model.reuse_kv_cache)."""
    from transformers import CLIPImageProcessor, LlamaTokenizer
    tokenizer = _attach_image_tokens(LlamaTokenizer.from_pretrained(visualcla_model or lora_model))
    if visualcla_model is not None:
        logger.info("Init VisualCLA model from pretrained")
        model = VisualCLAModel.from_merged_pretrained(visualcla_model, torch_dtype=torch_dtype, default_device=default_device,
                                                      device_map=device_map, load_in_8bit=load_in_8bit, **engine_kwargs)
    else:
        assert text_model is not None and vision_model is not None
        logger.info("Init VisualCLA model with pretrained text/image encoders")
        model = VisualCLAModel.from_vision_text_pretrained(vision_model, text_model, visualcla_config=VisualCLAConfig.from_pretrained(lora_model),
                                                           torch_dtype=torch_dtype, default_device=default_device,
                                                           device_map=device_map, load_in_8bit=load_in_8bit, **engine_kwargs)
    if os.environ.get("VCLA_GPU_PREPROCESS", "") not in ("", "0"):
        # opt-in: same pre-processing (Pillow-exact) on the device, pixel_values never leave HBM (image_processing_vcla.py)
        from .image_processing_vcla import VclaImageProcessor
        image_processor = VclaImageProcessor.from_pretrained(vision_model or visualcla_model)
    else:
        image_processor = CLIPImageProcessor.from_pretrained(vision_model or visualcla_model)
    image_processor.patch_size = model.vision_model.config.patch_size
    model.tokenizer = tokenizer
    model.image_processor = image_processor
    model.image_at_head = False
    model.reuse_kv_cache = bool(reuse_kv_cache)
    nq = model.config.visual_resampler_config["num_query_tokens"]
    model.num_patch = nq if nq != -1 else (image_processor.size["shortest_edge"] // image_processor.patch_size) ** 2 + 1
    return model, tokenizer, image_processor


def _pixels(model, image):
    from PIL import Image
    if isinstance(image, str):
        return model.image_processor(Image.open(image), return_tensors="pt").pixel_values
    if isinstance(image, Image.Image):
        return model.image_processor(image, return_tensors="pt").pixel_values
    return image


def _prepare(model, image, text, history, generation_config):
    generation_config = generation_config or DEFAULT_GENERATION_CONFIG
    generation_config.bos_token_id = generation_config.bos_token_id or model.tokenizer.bos_token_id
    pixel_values = _pixels(model, image)
    enc = encoding_text(history, text, model.num_patch, model.tokenizer)
    # the reference feeds fp16 pixels on GPU (:159); the engine converts whatever arrives to its bf16 operand type
    enc["pixel_values"] = pixel_values.half()
    enc = enc.to(model.device)
    entry = {"type": "instruction", "value": text}
    if len(history) == 0:
        entry["first_instruction"] = True
    history.append(entry)
    return enc, generation_config


def _cache_kwargs(model):
    """With model.reuse_kv_cache, generate() gets the previous turn's KV-cache handle: the conversation so far is a prefix of
    this turn's prompt, so only the new instruction is prefilled and the image is not encoded again.  Off by default: the
    cached prefix's K/V came from the decode GEMMs, equal to a fresh prefill only within bf16 rounding, so a sampled reply can
    differ from the one without reuse under the same seed."""
    if not getattr(model, "reuse_kv_cache", False):
        return {}
    return dict(past_key_values=getattr(model, "_chat_kv_cache", None), return_dict_in_generate=True)


def _keep_cache(model, outputs):
    if not getattr(model, "reuse_kv_cache", False):
        return outputs
    model._chat_kv_cache = outputs.past_key_values
    return outputs.sequences


@torch.inference_mode()
def chat(model, image, text: str, history=[], generation_config=None):
    """ref: modeling_utils.py:143-178 (same mutable-default `history` contract as the reference)."""
    enc, generation_config = _prepare(model, image, text, history, generation_config)
    outputs = model.generate(input_ids=enc.input_ids, attention_mask=enc.attention_mask, pixel_values=enc.pixel_values,
                             generation_config=generation_config, **_cache_kwargs(model))
    outputs = _keep_cache(model, outputs)
    response = model.tokenizer.decode(outputs[0], skip_special_tokens=True)
    history.append({"type": "response", "value": response})
    print("Response:", response)
    print("History:", history)
    return response, history


class Stream:
    """Stopping-criteria shaped callback: called after every generated token with the ids so far (ref :404-411)."""

    def __init__(self, callback_func=None):
        self.callback_func = callback_func

    def __call__(self, input_ids, scores) -> bool:
        if self.callback_func is not None:
            try:
                self.callback_func(input_ids[0])
            except StopIteration:
                # the consumer stopped listening (Iteratorize left its `with` block): end generation normally, so that
                # generate() still returns -- with reuse_kv_cache, its cache handle records the tokens fed so far
                return True
        return False


class Iteratorize:
    """Run `func(callback=..., **kwargs)` on a worker thread and iterate over what it passes to the callback
    (ref :415-472).  Leaving the `with` block stops generation at the next token and waits for the worker to finish, so the
    model is idle (and a chat turn's cache handle stored) when the block is left."""

    _END = object()

    def __init__(self, func, kwargs=None, callback=None):
        self._q: "queue.Queue" = queue.Queue()
        self._stop = threading.Event()
        self._done_cb = callback

        def on_token(val):
            if self._stop.is_set():
                raise StopIteration
            self._q.put(val)

        def work():
            ret = None
            try:
                ret = func(callback=on_token, **(kwargs or {}))
            except StopIteration:
                pass
            except Exception:  # the reference swallows worker exceptions too (:438-444)
                logger.exception("generation thread failed")
            clear_torch_cache()
            self._q.put(self._END)
            if self._done_cb:
                self._done_cb(ret)

        self._thread = threading.Thread(target=work, daemon=True)
        self._thread.start()

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get(True, None)
        if item is self._END:
            raise StopIteration
        return item

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self._stop.set()
        if self._thread is not threading.current_thread():
            self._thread.join()
        clear_torch_cache()


@torch.inference_mode()
def chat_in_stream(model, image, text: str, history=[], generation_config=None):
    """Generator of (response_so_far, history) (ref: modeling_utils.py:180-247).  Its only stopping criterion is a Stream, so generate()
    runs it on the device decode graphs with each token published as it is chosen: under the same seed it ends on chat()'s reply."""
    enc, generation_config = _prepare(model, image, text, history, generation_config)
    eos_token_id = model.tokenizer.eos_token_id
    base_history = deepcopy(history)
    params = generation_config.to_dict()
    params.pop("transformers_version", None)
    gen_cfg = GenerationConfig(**params)

    def run(callback=None, **_):
        with torch.no_grad():
            out = model.generate(input_ids=enc.input_ids, attention_mask=enc.attention_mask, pixel_values=enc.pixel_values,
                                 generation_config=gen_cfg, stopping_criteria=[Stream(callback_func=callback)], **_cache_kwargs(model))
            _keep_cache(model, out)

    response, hist = "", history
    with Iteratorize(run) as stream:
        for ids in stream:
            if len(ids) and int(ids[-1]) == eos_token_id:
                # prompt lookup decoding publishes several tokens per step: the ones before the EOS are still part of the reply
                if len(ids) > 1 and model.tokenizer.decode(ids[:-1], skip_special_tokens=True) != response:
                    response = model.tokenizer.decode(ids[:-1], skip_special_tokens=True)
                    hist = deepcopy(base_history)
                    hist.append({"type": "response", "value": response})
                    yield response, hist
                break
            response = model.tokenizer.decode(ids, skip_special_tokens=True)
            hist = deepcopy(base_history)
            hist.append({"type": "response", "value": response})
            yield response, hist
    print("Response:", response)
    print("History:", hist)


# --------------------------------------------------------------------------------------------------
# extra samplers exposed by the reference (TFS / Top-A / Mirostat, ref :250-383) -- host-side torch ops on the
# logits the engine returns; the greedy path never touches them.
# --------------------------------------------------------------------------------------------------
class TailFreeLogitsWarper(LogitsProcessor):
    """Tail-free sampling: drop the tokens after the point where the cumulative |second derivative| of the
    sorted probabilities exceeds `tfs`."""

    def __init__(self, tfs: float, filter_value: float = -float("inf"), min_tokens_to_keep: int = 1):
        tfs = float(tfs)
        if not 0.0 <= tfs <= 1.0:
            raise ValueError(f"`tfs` has to be a float >= 0 and <= 1, but is {tfs}")
        self.tfs, self.filter_value, self.min_tokens_to_keep = tfs, filter_value, min_tokens_to_keep

    def __call__(self, input_ids, scores):
        s, order = torch.sort(scores, descending=True)
        p = s.softmax(-1)
        curv = p.diff().diff().abs()
        curv = curv / curv.sum(-1, keepdim=True)
        cdf = curv.cumsum(-1)
        drop = cdf > self.tfs
        # the two diffs shorten the axis by 2: always keep the head token, always drop the last one
        drop = torch.cat([torch.zeros_like(drop[:, :1]), drop, torch.ones_like(drop[:, :1])], dim=-1)
        if self.min_tokens_to_keep > 1:
            drop[:, : self.min_tokens_to_keep] = False
        mask = drop.scatter(1, order, drop)
        return scores.masked_fill(mask, self.filter_value)


class TopALogitsWarper(LogitsProcessor):
    """Top-A: drop tokens whose probability is below top_a * p_max^2."""

    def __init__(self, top_a: float, filter_value: float = -float("inf"), min_tokens_to_keep: int = 1):
        top_a = float(top_a)
        if not 0.0 <= top_a <= 1.0:
            raise ValueError(f"`top_a` has to be a float >= 0 and <= 1, but is {top_a}")
        self.top_a, self.filter_value, self.min_tokens_to_keep = top_a, filter_value, min_tokens_to_keep

    def __call__(self, input_ids, scores):
        s, order = torch.sort(scores, descending=True)
        p = s.softmax(-1)
        drop = p < (p[:, :1] ** 2) * self.top_a
        if self.min_tokens_to_keep > 1:
            drop[:, : self.min_tokens_to_keep] = False
        mask = drop.scatter(1, order, drop)
        return scores.masked_fill(mask, self.filter_value)


class MirostatLogitsWarper(LogitsProcessor):
    """Mirostat v2 (batch element 0, like the reference): truncate to surprise < mu, sample, adapt mu."""

    def __init__(self, mirostat_mode: int, mirostat_tau: float, mirostat_eta: float, filter_value: float = -float("inf"),
                 min_tokens_to_keep: int = 1):
        if mirostat_mode not in (2,):
            raise ValueError(f"`mirostat` has to be a an integer 2, but is {mirostat_mode}")
        self.tau, self.eta, self.mu = mirostat_tau, mirostat_eta, 2 * mirostat_tau
        self.filter_value, self.min_tokens_to_keep = filter_value, min_tokens_to_keep

    def __call__(self, input_ids, scores):
        row = scores[0]
        s, order = torch.sort(row, descending=True)
        p = s.softmax(-1)
        surprise = -torch.log2(p)
        keep = int((surprise <= self.mu).sum().clamp(min=1))
        p = torch.softmax(s[:keep], dim=0)
        pick = torch.multinomial(p, 1)
        self.mu -= self.eta * (float(-torch.log2(p[pick])) - self.tau)
        out = torch.full_like(scores, self.filter_value)
        out[0, order[pick]] = 0.0
        return out


def hijack_samplers():
    """ref: modeling_utils.py:395-400 teaches GenerationConfig the extra knobs.  transformers >= 4.4x keeps unknown
    GenerationConfig kwargs as attributes already, so only defaults are registered here; VisualCLAModel.generate
    reads `tfs` / `top_a` when present."""
    for name, default in (("tfs", 1.0), ("top_a", 0.0), ("mirostat_mode", 0), ("mirostat_eta", 0.1), ("mirostat_tau", 5)):
        if not hasattr(GenerationConfig, name):
            setattr(GenerationConfig, name, default)


def clear_torch_cache():
    gc.collect()
    if torch.cuda.device_count() > 0:
        torch.cuda.empty_cache()
