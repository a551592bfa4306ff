"""VisualCLAModel on the H100-native path.

Same public surface as the reference's composite model (ref: models/visualcla/modeling_visualcla.py:70-404):
`from_pretrained / from_merged_pretrained / from_vision_text_pretrained`, `forward`, `generate`,
`get/set_{input,output}_embeddings`, the attributes the reference's callers read (`.tokenizer`,
`.image_processor`, `.num_patch`, `.image_at_head`, `.device`, `.config`, `.text_model`, `.vision_model`,
`.visual_resampler`, `.image_projection_layer`) and the nn.Module verbs they use (`.eval() .float() .half()
.to() .state_dict() .resize_token_embeddings()`).  Underneath there are no nn.Modules: all arithmetic runs in
hand-written sm_90a kernels behind the C ABI in include/vcla.h (see engine.py / _native.py).
"""
from __future__ import annotations

import contextlib
import copy
import glob
import json
import os
import weakref
from types import SimpleNamespace
from typing import Dict, List, NamedTuple, Optional, Tuple, Union

import torch

from . import _native as N
from .configuration_visualcla import VisualCLAConfig
from .engine import Engine, kv_format_of, path_config_7b


# --------------------------------------------------------------------------------------------------
# checkpoint shards
# --------------------------------------------------------------------------------------------------
def _iter_checkpoint(directory: str):
    """Yield (name, tensor) from every `pytorch_model*.bin` / `*.safetensors` shard of an HF-style directory."""
    files = sorted(glob.glob(os.path.join(directory, "pytorch_model*.bin"))) + \
        sorted(glob.glob(os.path.join(directory, "*.safetensors")))
    if not files:
        raise ValueError(f"no checkpoint shards (pytorch_model*.bin / *.safetensors) under {directory}")
    for f in files:
        if f.endswith(".safetensors"):
            from safetensors.torch import load_file
            sd = load_file(f, device="cpu")
        else:
            sd = torch.load(f, map_location="cpu", weights_only=True)
        for k, v in sd.items():
            yield k, v
        del sd


class _EmbeddingView:
    """What `get_input_embeddings()` / `get_output_embeddings()` return: `.weight` materialises the table."""

    def __init__(self, model: "VisualCLAModel", name: str):
        self._model, self._name = model, name

    @property
    def weight(self) -> torch.Tensor:
        return self._model._engine.read_weight(self._name).to(self._model.device)

    def __call__(self, input_ids: torch.Tensor) -> torch.Tensor:
        return torch.nn.functional.embedding(input_ids.to(self._model.device), self.weight)


class _SubModel:
    """Lightweight handle standing in for the reference's nn.Module children (only what callers touch)."""

    def __init__(self, model: "VisualCLAModel", prefix: str, config):
        self._model, self._prefix = model, prefix
        self.config = config

    def state_dict(self) -> Dict[str, torch.Tensor]:
        return {k[len(self._prefix):]: v for k, v in self._model.state_dict().items() if k.startswith(self._prefix)}

    def get_input_embeddings(self):
        return self._model.get_input_embeddings()

    def get_output_embeddings(self):
        return self._model.get_output_embeddings()


class VclaKVCache:
    """What `generate(..., return_dict_in_generate=True).past_key_values` holds: a handle on the engine's resident KV cache, not the
    tensors.  It records the token ids that are really in the cache (the prompt, then every token fed to a decode step -- with EOS
    on the device that includes the pad steps run past EOS, never the last, unfed pick), the layout and a device copy of the pixels.
    Passing it back with the whole conversation as `input_ids` (as with HF's `past_key_values`) lets generate() keep the longest
    common prefix and prefill only the rest.  Any later prefill, decode, reset or weight change on the engine makes it stale, and a
    stale handle simply means a full prefill."""

    def __init__(self, engine, session: int, ids: Optional[torch.Tensor], mode: int, pixel_values: Optional[torch.Tensor]):
        self._engine = weakref.ref(engine)
        self.session = session
        self.ids = ids                      # (L,) int64 on the CPU, or None when the cache cannot be reused (batch > 1, padding)
        self.mode = mode
        self.pixel_values = pixel_values

    def is_current(self, engine) -> bool:
        return self._engine() is engine and getattr(engine, "session", None) == self.session

    def __len__(self):
        return 0 if self.ids is None else int(self.ids.numel())


class _DevicePlan(NamedTuple):
    """how a generate() call runs on the decode graphs (VisualCLAModel._device_plan)"""
    spec: Optional["N.VclaSampler"]     # the device sampler, or None: the argmax graphs
    lookup: Optional[Tuple[int, int]]   # prompt lookup decoding's (k, n), or None
    streamed: bool                      # tokens reach a streamer / Stream criteria through the ring as they are chosen


class VisualCLAModel:
    config_class = VisualCLAConfig
    base_model_prefix = "visualcla"
    reuse_kv_cache = False     # chat() / chat_in_stream(): keep the KV cache between turns (opt-in, see modeling_utils.chat)

    def __init__(self, config: VisualCLAConfig = None, vision_model=None, text_model=None, device=None,
                 max_batch: int = 8, max_seq: int = 1024, max_prefill_tokens: Optional[int] = None,
                 torch_dtype=torch.bfloat16, load_in_8bit: bool = False, kv_cache_dtype=None):
        if config is None:
            raise ValueError("VisualCLAModel needs a VisualCLAConfig")
        if vision_model is not None or text_model is not None:
            raise NotImplementedError("pre-built nn.Module sub-models are not used on the H100 path; load weights with "
                                      "from_merged_pretrained / from_vision_text_pretrained / load_state_dict")
        self.config = config
        # load_in_8bit: the seven LLaMA projections of every layer become weight-only int8 with per-row scales (what bitsandbytes
        # converts in the reference, modeling_visualcla.py:151-156); everything else stays as it is
        self._engine = Engine(config.to_path_config(), max_batch=max_batch, max_seq=max_seq, max_prefill_tokens=max_prefill_tokens,
                              device=device, weight_format=Engine.WEIGHT_INT8 if load_in_8bit else Engine.WEIGHT_BF16,
                              kv_format=kv_format_of(kv_cache_dtype))
        self.dtype = torch.bfloat16      # compute dtype of the path (bf16 operands, fp32 accumulate / residual stream)
        self.requested_dtype = torch_dtype
        self.image_at_head = True        # constructor default of the reference (:108); the loader flips it (:134)
        self.tokenizer = None
        self.image_processor = None
        self.num_patch = self._engine.nq
        self.vision_embed_dim = config.vision_config["hidden_size"]
        self.text_embed_dim = config.text_config["hidden_size"]
        self.text_model = _SubModel(self, "text_model.", SimpleNamespace(**config.text_config))
        self.vision_model = _SubModel(self, "vision_model.", SimpleNamespace(**config.vision_config))
        self.visual_resampler = _SubModel(self, "visual_resampler.", SimpleNamespace(**(config.visual_resampler_config or {})))
        self.image_projection_layer = _SubModel(self, "image_projection_layer.", None)
        self.generation_config = None
        self._tok_buf = {}

    # ---- nn.Module-ish verbs used by the reference's scripts ------------------------------------
    @property
    def device(self) -> torch.device:
        return self._engine.device

    def eval(self): return self
    def float(self): return self
    def half(self): return self
    def bfloat16(self): return self
    def requires_grad_(self, *_a, **_k): return self
    def train(self, mode: bool = False):
        if mode:
            raise NotImplementedError("the H100 path is inference-only (the reference ships no training code)")
        return self

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (str, torch.device)) and torch.device(a).type != "cuda":
                raise N.NativeError("the H100 path has no CPU fallback: model.to('cpu') is not supported")
        return self

    def parameters(self):
        return iter(())

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Host copies of every tensor.  With load_in_8bit the int8 projections come back as fp32 q * s, so save_merged_pretrained writes
        them twice the size of bf16; loading that checkpoint with load_in_8bit=True quantises q * s again and reproduces q."""
        return {n: self._engine.read_weight(n) for n, _s, _k in self._engine.weight_table()}

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        loaded, unexpected = self._engine.load_state_dict(sd)
        expected = {n for n, _s, _k in self._engine.weight_table()}
        missing = sorted(expected - loaded)
        # tolerated extras: the dead pooler (ref: modeling_visual_resampler.py:725) and position_ids buffers
        unexpected = [k for k in unexpected if "pooler" not in k and "position_ids" not in k and "rotary_emb.inv_freq" not in k]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing {missing[:5]}... ({len(missing)}), unexpected {unexpected[:5]}... ({len(unexpected)})")
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def get_input_embeddings(self): return _EmbeddingView(self, "text_model.model.embed_tokens.weight")
    def get_output_embeddings(self): return _EmbeddingView(self, "text_model.lm_head.weight")
    def set_input_embeddings(self, new): self._engine.load_weight("text_model.model.embed_tokens.weight", new.weight)
    def set_output_embeddings(self, new): self._engine.load_weight("text_model.lm_head.weight", new.weight)

    def resize_token_embeddings(self, new_num_tokens: Optional[int] = None):
        """ref: scripts/inference/inference.py:69 -- grow the vocab (49954 -> 49958) before LoRA weights are applied."""
        old = self._engine.vocab
        if new_num_tokens is None or new_num_tokens == old:
            return self.get_input_embeddings()
        e = self._engine
        q8 = [n for n, _s, kind in e.weight_table() if kind == 2]
        sd = {n: e.read_weight(n) for n, _s, kind in e.weight_table() if kind != 2}
        cfg = copy.deepcopy(self.config)
        cfg.text_config["vocab_size"] = int(new_num_tokens)
        new = Engine(cfg.to_path_config(), max_batch=e.max_batch, max_seq=e.max_seq, max_prefill_tokens=e.max_prefill_tokens, device=e.device,
                     weight_format=e.weight_format, kv_format=e.kv_format)
        for n in q8:                        # int8 tensors move as stored (quantising q * s again could change them)
            new.load_weight_q8(n, *e.read_weight_q8(n))
        for k in ("text_model.model.embed_tokens.weight", "text_model.lm_head.weight"):
            w = sd.pop(k).float()
            grown = torch.zeros(new_num_tokens, w.shape[1])
            n = min(old, new_num_tokens)
            grown[:n] = w[:n]
            if new_num_tokens > old:
                grown[old:] = w[:old].mean(0, keepdim=True)     # HF initialises new rows from the mean embedding
            new.load_weight(k, grown)
        new.load_state_dict(sd)
        e.close()
        self._engine, self.config = new, cfg
        self.text_model.config = SimpleNamespace(**cfg.text_config)
        self._tok_buf = {}
        return self.get_input_embeddings()

    @property
    def kv_cache_dtype(self) -> torch.dtype:
        """Storage of the KV cache: torch.int8 (int8 rows + one fp32 scale per token and head, kv_cache_dtype="int8") or torch.bfloat16."""
        return torch.int8 if self._engine.kv_format == Engine.KV_INT8 else torch.bfloat16

    # ---- constructors -----------------------------------------------------------------------------
    @classmethod
    def from_synthetic(cls, path_cfg: Union[str, Dict] = "7b", seed: int = 0, **kw) -> "VisualCLAModel":
        """Random-init weights of the given architecture, generated on the device (no checkpoint files offline)."""
        p = path_config_7b() if path_cfg == "7b" else dict(path_cfg)
        model = cls(VisualCLAConfig.from_path_config(p), **kw)
        model._engine.init_synthetic(seed)
        return model

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, *args, **kwargs) -> "VisualCLAModel":
        """ref: modeling_visualcla.py:110-118.  Accepts a merged directory (text_encoder/ + vision_encoder/ +
        pytorch_model.bin) or a flat HF directory holding the whole composite state dict."""
        path = pretrained_model_name_or_path
        if not os.path.isdir(path):
            raise ValueError(f"{path} is not a local directory (no network access on this path)")
        kw = dict(torch_dtype=kwargs.pop("torch_dtype", torch.bfloat16), default_device=kwargs.pop("default_device", None),
                  device_map=kwargs.pop("device_map", None), load_in_8bit=kwargs.pop("load_in_8bit", False))
        kwargs.pop("_fast_init", None)
        if os.path.isdir(os.path.join(path, "text_encoder")):
            return cls.from_merged_pretrained(path, **kw, **kwargs)
        config = VisualCLAConfig.from_pretrained(path)
        model = cls(config, device=kw["default_device"], torch_dtype=kw["torch_dtype"], load_in_8bit=kw["load_in_8bit"], **kwargs)
        model.load_state_dict(dict(_iter_checkpoint(path)))
        return model

    @classmethod
    def from_merged_pretrained(cls, visualcla_model_name_or_path: str = None, *args, **kwargs) -> "VisualCLAModel":
        """ref: modeling_visualcla.py:120-181.  The four kwargs are REQUIRED there (popped without default); same here."""
        path = visualcla_model_name_or_path
        if not os.path.isdir(path):
            raise ValueError(f"{path} is not a local directory (the reference's hub path is broken too, SURVEY 3.6)")
        torch_dtype = kwargs.pop("torch_dtype")
        default_device = kwargs.pop("default_device")
        _device_map = kwargs.pop("device_map")          # whole model lives on one GPU (14.5 GB of 180 GB); DP replicates it
        load_in_8bit = kwargs.pop("load_in_8bit")
        config = VisualCLAConfig.from_pretrained(path)
        text_dir, vision_dir = os.path.join(path, "text_encoder"), os.path.join(path, "vision_encoder")
        with open(os.path.join(text_dir, "config.json")) as f:
            config.text_config = json.load(f)
        with open(os.path.join(vision_dir, "config.json")) as f:
            vc = json.load(f)
            config.vision_config = vc.get("vision_config", vc) if "hidden_size" not in vc else vc
        model = cls(config, device=default_device, torch_dtype=torch_dtype, load_in_8bit=bool(load_in_8bit), **kwargs)
        eng = model._engine
        seen = set()
        for k, v in _iter_checkpoint(text_dir):
            if "rotary_emb.inv_freq" in k:
                continue
            eng.load_weight("text_model." + k, v); seen.add("text_model." + k)
        for k, v in _iter_checkpoint(vision_dir):
            if "position_ids" in k:
                continue
            eng.load_weight("vision_model." + k, v); seen.add("vision_model." + k)
        for k, v in _iter_checkpoint(path):
            if k.startswith("visual_resampler.") and "pooler" not in k or k.startswith("image_projection_layer."):
                eng.load_weight(k, v); seen.add(k)
        missing = sorted({n for n, _s, _k in eng.weight_table()} - seen)
        if missing:
            raise RuntimeError(f"merged checkpoint {path} lacks {len(missing)} tensors, e.g. {missing[:4]}")
        return model

    @classmethod
    def from_vision_text_pretrained(cls, vision_model_name_or_path: str = None, text_model_name_or_path: str = None,
                                    visualcla_config: Union[str, VisualCLAConfig] = None, torch_dtype=torch.float16,
                                    default_device=None, device_map=None, load_in_8bit=False, **kwargs) -> "VisualCLAModel":
        """ref: modeling_visualcla.py:183-261: base CLIP + base LLaMA, resampler/projector randomly initialised
        (the LoRA path then overwrites them; LoRA folding itself is a 'next' row, SURVEY 8f-2)."""
        if vision_model_name_or_path is None:
            raise ValueError("If `vision_model` is not defined as an argument, a `vision_model_name_or_path` has to be defined")
        if text_model_name_or_path is None:
            raise ValueError("If `text_model` is not defined as an argument, a `text_model_name_or_path` has to be defined")
        if isinstance(visualcla_config, str):
            visualcla_config = VisualCLAConfig.from_pretrained(visualcla_config)
        config = copy.deepcopy(visualcla_config)
        with open(os.path.join(text_model_name_or_path, "config.json")) as f:
            config.text_config = json.load(f)
        with open(os.path.join(vision_model_name_or_path, "config.json")) as f:
            vc = json.load(f)
            config.vision_config = vc.get("vision_config", vc) if "hidden_size" not in vc else vc
        model = cls(config, device=default_device, torch_dtype=torch_dtype, load_in_8bit=bool(load_in_8bit), **kwargs)
        eng = model._engine
        eng.init_synthetic(0)   # resampler + projector: fresh init, as in the reference
        known = {n for n, _s, _k in eng.weight_table()}
        seen = set()
        for k, v in _iter_checkpoint(text_model_name_or_path):
            if "rotary_emb.inv_freq" not in k:
                eng.load_weight("text_model." + k, v); seen.add("text_model." + k)
        for k, v in _iter_checkpoint(vision_model_name_or_path):
            # a full CLIPModel checkpoint also carries the text tower / projections: only the vision tower is on the path
            name = "vision_model." + k
            if name in known:
                eng.load_weight(name, v); seen.add(name)
        # only the resampler and the projector may keep their fresh initialisation: a missing shard or a renamed key must
        # not leave LLaMA / CLIP layers at random weights
        missing = sorted(n for n in known - seen if n.startswith(("text_model.", "vision_model.")))
        if missing:
            raise RuntimeError(f"base checkpoints lack {len(missing)} tensors of the text/vision towers, e.g. {missing[:4]}")
        return model

    def save_merged_pretrained(self, output_dir: str):
        """Write the merged-directory layout of ref: scripts/merge_llama_with_visualcla_lora.py:87-97."""
        os.makedirs(os.path.join(output_dir, "text_encoder"), exist_ok=True)
        os.makedirs(os.path.join(output_dir, "vision_encoder"), exist_ok=True)
        sd = self.state_dict()
        text = {k[len("text_model."):]: v for k, v in sd.items() if k.startswith("text_model.")}
        vision = {k[len("vision_model."):]: v for k, v in sd.items() if k.startswith("vision_model.")}
        rest = {k: v for k, v in sd.items() if not k.startswith(("text_model.", "vision_model."))}
        torch.save(text, os.path.join(output_dir, "text_encoder", "pytorch_model.bin"))
        torch.save(vision, os.path.join(output_dir, "vision_encoder", "pytorch_model.bin"))
        torch.save(rest, os.path.join(output_dir, "pytorch_model.bin"))
        with open(os.path.join(output_dir, "text_encoder", "config.json"), "w") as f:
            json.dump(self.config.text_config, f)
        with open(os.path.join(output_dir, "vision_encoder", "config.json"), "w") as f:
            json.dump(self.config.vision_config, f)
        self.config.save_pretrained(output_dir)

    @torch.no_grad()
    def embed_images(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """pixels (N,3,I,I) -> image embeddings (N, num_query_tokens, text_hidden): the tg-webui pipeline's entry point
        (ref: scripts/inference/text_generation_webui/visualcla/visualcla.py:116-129)."""
        return self._engine.vision_encode(pixel_values, return_embeds=True)

    # ---- prompt assembly (host side of ref :290-312 / :356-377) -----------------------------------
    def _image_layout(self, input_ids: torch.Tensor, pixel_values):
        """-> (image_mode, img_rows or None).  Replicates the reference's per-sample checks for the placeholder layout."""
        if pixel_values is None:
            return N.TEXT_ONLY, None
        if self.image_at_head:
            return N.IMAGE_AT_HEAD, None
        tok = self.tokenizer
        if tok is None:
            raise AttributeError("model.tokenizer (img_start_token_id / img_end_token_id) is required when image_at_head is False")
        ids = input_ids.detach().cpu()
        nq = self._engine.nq
        rows = []
        for cur in ids:
            pos = torch.where(cur == tok.img_start_token_id)[0]
            if len(pos) == 0:
                rows.append(-1)
                continue
            p = int(pos[0])
            if p + nq + 1 >= cur.shape[0] or int(cur[p + nq + 1]) != tok.img_end_token_id:
                raise ValueError(f"Num of patch ({nq}) is not equal to the length of pre-filled image patch tokens.")
            rows.append(p + 1)
        return N.IMAGE_PLACEHOLDER, torch.tensor(rows, dtype=torch.int32)

    def _left_pad(self, attention_mask, image_mode):
        """attention_mask -> per-sequence left-padding counts (or None).  HF batches prompts of different lengths by LEFT
        padding; any other mask shape is rejected."""
        if attention_mask is None or bool((attention_mask != 0).all()):
            return None
        m = (attention_mask != 0).to("cpu")
        pads = (~m).sum(1)
        T = m.shape[1]
        expect = torch.arange(T)[None, :] >= pads[:, None]
        if not torch.equal(m, expect):
            raise NotImplementedError("only left padding (attention_mask = [0]*p + [1]*(T-p)) is supported on the H100 path")
        if bool((pads >= T).any()):
            raise ValueError("attention_mask masks a whole sequence")
        if image_mode == N.IMAGE_AT_HEAD:
            raise NotImplementedError("padded batches need the placeholder layout (image_at_head=False): the reference's at-head splice "
                                      "ignores the mask (ref modeling_visualcla.py:291)")
        return pads.to(torch.int32)

    # ---- forward: logits for every position (ref :264-330) ---------------------------------------
    @torch.no_grad()
    def forward(self, input_ids=None, pixel_values=None, attention_mask=None, position_ids=None, past_key_values=None,
                labels=None, use_cache=None, return_loss=None, return_dict=None, **kwargs):
        from transformers.modeling_outputs import CausalLMOutputWithPast
        if past_key_values is not None:
            raise NotImplementedError("forward(past_key_values=...) is not supported; use generate()")
        mode, rows = self._image_layout(input_ids, pixel_values)
        pads = self._left_pad(attention_mask, mode)
        eng = self._engine
        if mode != N.TEXT_ONLY:
            if mode == N.IMAGE_AT_HEAD and labels is None:
                # ref quirk (:313-315): labels[:, [0]] is indexed unconditionally in this layout
                raise TypeError("'NoneType' object is not subscriptable (labels are required with image_at_head=True)")
            eng.vision_encode(pixel_values)
        _, _, logits = eng.prefill(input_ids, mode, rows, all_logits=True, last_logits=False, left_pad=pads, pos_from_mask=False)
        loss = None
        if labels is not None:
            lab = labels.to(logits.device)
            if mode == N.IMAGE_AT_HEAD:
                fill = torch.full((lab.shape[0], eng.nq), -100, dtype=lab.dtype, device=lab.device)
                lab = torch.cat([lab[:, :1], fill, lab[:, 1:]], dim=1)
            loss = torch.nn.functional.cross_entropy(logits[:, :-1].reshape(-1, logits.shape[-1]).float(), lab[:, 1:].reshape(-1), ignore_index=-100)
        if return_dict is False:
            return ((loss,) if loss is not None else ()) + (logits,)
        return CausalLMOutputWithPast(loss=loss, logits=logits)

    __call__ = forward

    # ---- generate: only the NEW tokens are returned (ref :333-392, SURVEY 3.6) --------------------
    def _resolve_generation_config(self, generation_config, kwargs):
        from transformers import GenerationConfig
        gc = copy.deepcopy(generation_config) if generation_config is not None else GenerationConfig()
        unused = gc.update(**kwargs)
        for k in list(unused):
            if k in ("output_scores", "output_logits", "return_dict_in_generate", "use_cache", "tfs", "top_a", "mirostat_mode", "mirostat_tau", "mirostat_eta"):
                setattr(gc, k, unused.pop(k))
        if unused:
            raise ValueError(f"generate(): unsupported arguments {sorted(unused)}")
        beams = getattr(gc, "num_beams", 1) or 1
        nrs = getattr(gc, "num_return_sequences", 1) or 1
        if beams > 1 and nrs > beams:
            raise ValueError(f"`num_return_sequences` ({nrs}) has to be smaller or equal to `num_beams` ({beams}).")
        # without beams, num_return_sequences > 1 reaches generate() only with do_sample=True (GenerationConfig refuses greedy)
        return gc

    @staticmethod
    def _eos_set(gc):
        e = gc.eos_token_id
        if e is None:
            return []
        return [int(x) for x in (e if isinstance(e, (list, tuple)) else [e])]

    @torch.no_grad()
    def generate(self, input_ids=None, pixel_values=None, attention_mask=None, generation_config=None,
                 logits_processor=None, stopping_criteria=None, prefix_allowed_tokens_fn=None, synced_gpus=False, **kwargs):
        """HF generate() over the device path; returns the new tokens only.  do_sample=True with num_return_sequences=N > 1 returns
        B * N rows, row b * N + j being reply j of prompt b (HF's repeat_interleave order): each prompt is encoded and prefilled once
        and its KV pages are shared by its N rows, which then decode as a batch, each with its own draws.  prompt_lookup_num_tokens is
        ignored then, as for any batch above one row (HF refuses assisted generation with num_return_sequences > 1)."""
        past_key_values = kwargs.pop("past_key_values", None)
        streamer = kwargs.pop("streamer", None)
        gc = self._resolve_generation_config(generation_config, kwargs)
        if prefix_allowed_tokens_fn is not None:
            raise NotImplementedError("prefix_allowed_tokens_fn is not supported on the H100 path")
        if (getattr(gc, "num_beams", 1) or 1) > 1:
            return self._generate_beams(gc, input_ids, pixel_values, attention_mask, logits_processor, stopping_criteria, streamer)
        eng = self._engine
        B = input_ids.shape[0]
        n_ret = int(getattr(gc, "num_return_sequences", 1) or 1)     # > 1 only when sampling: rows b * n_ret + j, forked per prompt
        per_call = eng.max_batch
        if n_ret > 1:
            cap = min(eng.max_batch, 64)
            if n_ret > cap:
                raise NotImplementedError(f"num_return_sequences={n_ret} exceeds this model instance (at most min(max_batch, 64) = {cap} rows)")
            per_call = cap // n_ret
        if B > per_call:
            if streamer is not None:
                if n_ret > 1:
                    raise NotImplementedError(f"streaming {B} prompts x {n_ret} return sequences above {per_call * n_ret} rows is not supported")
                raise NotImplementedError(f"streaming a batch of {B} > max_batch={eng.max_batch} prompts is not supported")
            outs = []
            for s in range(0, B, per_call):
                sl = slice(s, s + per_call)
                outs.append(self.generate(input_ids[sl], None if pixel_values is None else pixel_values[sl],
                                          None if attention_mask is None else attention_mask[sl],
                                          gc, logits_processor, stopping_criteria, None, synced_gpus))
            width = max(o.shape[1] for o in outs)
            pad = gc.pad_token_id if gc.pad_token_id is not None else 0
            outs = [torch.nn.functional.pad(o, (0, width - o.shape[1]), value=pad) for o in outs]
            return torch.cat(outs, 0)

        mode, rows = self._image_layout(input_ids, pixel_values)
        pads = self._left_pad(attention_mask, mode)
        S = input_ids.shape[1] + (eng.nq if mode == N.IMAGE_AT_HEAD else 0)
        max_new = gc.max_new_tokens if gc.max_new_tokens is not None else max(int(gc.max_length or 20), 1)
        min_new = int(getattr(gc, "min_new_tokens", 0) or 0)
        if S + max_new > eng.max_seq:
            raise ValueError(f"prompt ({S}) + max_new_tokens ({max_new}) exceeds the context capacity max_seq={eng.max_seq} "
                             f"of this model instance")
        eos = self._eos_set(gc)
        pad = gc.pad_token_id if gc.pad_token_id is not None else (eos[0] if eos else 0)
        processors = self._build_processors(gc, logits_processor)
        sampling = bool(gc.do_sample)
        need_logits = sampling or len(processors) > 0 or bool(getattr(gc, "output_logits", False) or getattr(gc, "output_scores", False))
        crit = list(stopping_criteria) if stopping_criteria is not None else []

        R = B * n_ret                                                  # decoded rows
        reuse = self._plan_kv_reuse(past_key_values, input_ids, pixel_values, mode, rows, pads) if n_ret == 1 else None
        if mode != N.TEXT_ONLY and reuse is None:
            eng.vision_encode(pixel_values)

        def start(want_last_logits):
            """prefill the prompt, or keep the reusable cached prefix and extend it by the rest -> (last logits (B, V), first pick (R,))"""
            if reuse is None:
                with self._fanout_mode(n_ret):
                    ll, first, _ = eng.prefill(input_ids, mode, rows, all_logits=False, last_logits=want_last_logits, left_pad=pads,
                                               pos_from_mask=True)
            else:
                keep, rest = reuse
                eng.truncate([keep])
                ll, first, _ = eng.extend(rest, all_logits=False, last_logits=want_last_logits)
            return ll, first

        def finish(result, fed, logits=None):
            """the return value; with return_dict_in_generate also the cache handle (prompt + the tokens fed to decode steps)"""
            if not getattr(gc, "return_dict_in_generate", False):
                return result
            ids = px = None
            if R == 1 and pads is None:       # only such a cache can be reused: keep its ids and pixels, nothing otherwise
                ids = torch.cat([input_ids[0].detach().to("cpu", torch.int64), fed[0].detach().to("cpu", torch.int64)])
                px = None if pixel_values is None else pixel_values.detach().to(eng.device).clone()
            cache = VclaKVCache(eng, getattr(eng, "session", 0), ids, mode, px)
            return SimpleNamespace(sequences=result, logits=logits, scores=None, past_key_values=cache)

        dev = eng.device
        key = (R, need_logits)
        if key not in self._tok_buf:
            # persistent step buffers (their addresses key the captured CUDA graph).  chat() runs under torch.inference_mode and
            # chat_in_stream's worker thread does not: allocate them as ordinary tensors so both may update them in place.
            with torch.inference_mode(False):
                self._tok_buf[key] = (torch.zeros(R, dtype=torch.int32, device=dev),
                                      torch.empty(R, eng.vocab, dtype=torch.float32, device=dev) if need_logits else None)
        tok, logits = self._tok_buf[key]

        plan = self._device_plan(gc, R, S, max_new, eos, pad, min_new, need_logits, logits_processor, processors, crit, streamer)
        if plan is not None:
            lookup = (input_ids[0], *plan.lookup, max_new) if plan.lookup else None
            if plan.streamed:
                return self._generate_streamed(plan.spec, lookup, start, finish, R, max_new, eos, tok, streamer, crit)
            return self._generate_graphs(plan.spec, lookup, start, finish, R, max_new, eos, tok)

        # the per-step host loop: HF logits processors / sampling / criteria on the logits of every step
        out = torch.full((R, max_new), pad, dtype=torch.int64, device=dev)
        all_logits: List[torch.Tensor] = []
        if streamer is not None:
            streamer.put(torch.empty(R, 0, dtype=torch.int64))    # HF generate: put(input_ids) first -- none with inputs_embeds
        last, first_tok = start(need_logits)
        if n_ret > 1 and last is not None:
            last = last.repeat_interleave(n_ret, dim=0)          # the first step scores each prompt's last logits once per reply
        finished = torch.zeros(R, dtype=torch.bool, device=dev)
        n_done = 0
        for step in range(max_new):
            if step == 0:
                cur_logits, greedy = last, first_tok
            else:
                eng.decode_step(tok, tok, logits)
                cur_logits, greedy = logits, tok
            if need_logits:
                if getattr(gc, "output_logits", False):
                    all_logits.append(cur_logits.clone())
                scores = cur_logits
                if processors:
                    scores = cur_logits.clone()
                    if eos and step < min_new:
                        scores[:, eos] = -float("inf")
                    hist = out[:, :step]
                    for p in processors:
                        scores = p(hist, scores)
                if sampling:
                    probs = torch.softmax(scores.float(), dim=-1)
                    nxt = torch.multinomial(probs, num_samples=1).squeeze(1)
                else:
                    nxt = scores.argmax(dim=-1)
                nxt = nxt.to(torch.int32)
            else:
                nxt = greedy
            if eos:
                nxt = torch.where(finished, torch.full_like(nxt, pad), nxt)
            out[:, step] = nxt
            if nxt.data_ptr() != tok.data_ptr():
                tok.copy_(nxt)
            n_done = step + 1
            stop = False
            if streamer is not None:
                streamer.put(nxt.to("cpu", torch.int64))
            if eos:
                is_eos = torch.zeros_like(finished)
                for e in eos:
                    is_eos |= nxt == e
                finished |= is_eos
                # host poll (one sync) only every 8 steps: sequences are independent, so running a few extra
                # steps past the last EOS cannot change any retained token (HF syncs every step).  A streamer sees every
                # step, so with one the loop stops where HF does.
                if (step & 7) == 7 or step == max_new - 1 or streamer is not None:
                    stop = bool(finished.all())
            if self._criteria_stop(crit, out[:, :n_done], cur_logits if need_logits else None) or stop:
                break
        if streamer is not None:
            streamer.end()
        # a finished row already holds pad after its EOS
        return finish(self._cut_at_eos(out[:, :n_done], eos), out[:, : n_done - 1], tuple(all_logits) if all_logits else None)

    def _device_plan(self, gc, B, S, max_new, eos, pad, min_new, need_logits, logits_processor, processors, crit, streamer):
        """-> how this call runs on the decode graphs, or None: the per-step host loop.  Plain greedy without EOS runs the argmax
        graphs; anything else needs a device sampler spec (_device_sampler_spec draws its seed).  A call with a streamer or only Stream
        criteria streams on the device when the engine has the token ring and the call would run there without its Stream criteria;
        any other criterion, or VCLA_HOST_SAMPLER=1, keeps it on the host loop (VCLA_HOST_SAMPLER=1 leaves a non-streamed plain greedy
        call on the argmax graphs)."""
        from .modeling_utils import Stream
        stream_only = all(isinstance(c, Stream) for c in crit)
        streamed = streamer is not None or (len(crit) > 0 and stream_only)
        if streamed and (not stream_only or os.environ.get("VCLA_HOST_SAMPLER") == "1"
                         or not getattr(self._engine, "stream_supported", lambda: False)()):
            return None
        greedy = not need_logits and not eos and (streamed or not crit)
        spec = None
        if not (streamed and greedy):
            spec = self._device_sampler_spec(gc, eos, pad, min_new, logits_processor, [] if streamed else crit, processors)
            if spec is None and not greedy:
                return None
        k = self._lookup_tokens(gc, B, S, max_new)
        return _DevicePlan(spec, (k, int(getattr(gc, "max_matching_ngram_size", None) or 2)) if k else None, streamed)

    @staticmethod
    def _criteria_stop(crit, ids, scores) -> bool:
        """HF's stopping criteria on the tokens so far: every criterion runs; one returning a tensor stops only when all of it is True"""
        stop = False
        for cfn in crit:
            r = cfn(ids, scores)
            if isinstance(r, torch.Tensor):
                r = bool(r.all())
            stop = stop or bool(r)
        return stop

    # ---- the decode graphs: argmax, the device sampler, prompt lookup, each optionally streamed ------------------------------------
    @contextlib.contextmanager
    def _fanout_mode(self, n):
        """n > 1: the prefill inside forks every prompt to n rows (num_return_sequences); switched off again right after it"""
        if n > 1:
            self._engine.set_fanout(n)
        try:
            yield
        finally:
            if n > 1:
                self._engine.set_fanout(1)

    @contextlib.contextmanager
    def _sampler_mode(self, spec):
        """the device sampler (spec) for the prefill and decode steps inside, or the argmax graphs (None); always set before start()
        (the prefill picks the first token) and switched off last"""
        if spec is not None:
            self._engine.set_sampler(spec)
        try:
            yield
        finally:
            if spec is not None:
                self._engine.set_sampler(None)

    @contextlib.contextmanager
    def _decode_modes(self, start, tok, lookup=None, drain=None):
        """start() the call and put its first pick in tok.  drain given: the token ring is armed before the prefill, and on the way out
        drain() waits for the armed work still running before it is disarmed.  lookup = (prompt_ids, k, n, max_new) given: prompt
        lookup is set after the prefill (vcla_set_lookup refuses while an earlier call left more than one sequence resident) and unset
        after the ring is disarmed."""
        eng = self._engine
        if drain is not None:
            eng.stream_arm(True)
        try:
            _, first_tok = start(False)
            tok.copy_(first_tok)
            if lookup is not None:
                eng.set_lookup(*lookup)
            yield
        finally:
            if drain is not None:
                drain()
                eng.stream_arm(False)
            if lookup is not None:
                eng.set_lookup(None)

    def _decode_polled(self, tok, max_new, all_done):
        """graphs of 8 decode steps, one host poll of the per-row done flags (all_done()) between them, until every row is done or
        max_new tokens exist -> tokens decoded.  Rows are independent and a done row's tokens no longer change, so the steps run past
        the last one cannot change a retained token."""
        n_done = 1
        while n_done < max_new and not bool(all_done().bool().all()):
            k = min(8, max_new - n_done)
            self._engine.decode_many(tok, k)
            n_done += k
        return n_done

    def _generate_graphs(self, spec, lookup, start, finish, B, max_new, eos, tok):
        """generate() on the decode graphs with no host work per step.  Nothing can stop early: every step in one replay.  EOS: graphs of
        8 steps with a poll of the finished flags between them (a finished row only emits pad).  Prompt lookup: graphs of LOOKUP_CHUNK
        verification steps with a poll of the emitted count and the finished flag between them; each step emits the tokens one-token
        decoding would emit there, so the result, the EOS cut and the cache handle are those of the call without it."""
        eng = self._engine
        with self._sampler_mode(spec):
            with self._decode_modes(start, tok, lookup):
                if lookup is not None:
                    while True:
                        n_done, fin = eng.lookup_stats()[:2]
                        if n_done >= max_new or fin:
                            break
                        eng.decode_many(tok, self.LOOKUP_CHUNK)
                elif eos:
                    n_done = self._decode_polled(tok, max_new, lambda: eng.read_finished(B))
                else:
                    eng.decode_many(tok, max_new - 1)
                    n_done = max_new
            result = eng.read_history(B, n_done).t().to(torch.int64)
        # every history row was fed to a decode step except the last
        return finish(self._cut_at_eos(result, eos), result[:, : n_done - 1])

    # ---- streaming on the device: decode graphs publish every step into a pinned host ring (include/vcla.h, token streaming) ----
    STREAM_CHUNK = 8      # decode steps per graph replay while streaming

    def _generate_streamed(self, spec, lookup, start, finish, B, max_new, eos, tok, streamer, crit):
        """generate() with a streamer and / or Stream criteria, on the device: the graphs of _generate_graphs run armed, so the tokens
        reach the host through the ring as they are chosen.  HF's protocol: put an empty (B, 0) tensor first, then each batch of new
        tokens (int64, on the CPU) to streamer.put and then to the criteria, and end() last.  Launching stops at EOS, at max_new_tokens
        or when a criterion returns True; the steps still running then are drained and dropped."""
        if streamer is not None:
            streamer.put(torch.empty(B, 0, dtype=torch.int64))    # HF generate: put(input_ids) first -- none with inputs_embeds
        rows = torch.empty(B, max_new, dtype=torch.int64)         # host copy of the published tokens

        def publish(new, n_kept):
            """new tokens, already in rows[:, :n_kept] -> the streamer, then the criteria; True when a criterion stops the call"""
            if streamer is not None:
                streamer.put(new.clone())
            return self._criteria_stop(crit, rows[:, :n_kept], None)

        with self._sampler_mode(spec):
            if lookup is None:
                n_kept = self._stream_steps(start, tok, rows, max_new, eos, publish)
            else:
                n_kept = self._stream_lookup(start, tok, rows, max_new, eos, publish, lookup)
        if streamer is not None:
            streamer.end()
        # the device sampler already pads a finished row; the cache handle records the tokens fed up to the cut, and steps run past
        # it lie beyond its length
        return finish(rows[:, :n_kept].to(self._engine.device), rows[:, : n_kept - 1])

    def _stream_steps(self, start, tok, rows, max_new, eos, publish):
        """graphs of up to STREAM_CHUNK decode steps; the next one is enqueued once the second-to-last step of the running one is
        published, so the device never waits for the host.  One publish per step (HF _sample), so at most STREAM_CHUNK + 1 steps run
        past a stop.  -> tokens kept"""
        eng = self._engine
        B = rows.shape[0]
        eos_t = torch.tensor(eos, dtype=torch.int64) if eos else None
        finished = torch.zeros(B, dtype=torch.bool)
        n_launched = n_kept = 0

        def launch():
            nonlocal n_launched
            k = min(self.STREAM_CHUNK, max_new - n_launched)
            eng.decode_many(tok, k)
            n_launched += k

        with self._decode_modes(start, tok, drain=lambda: n_launched and eng.stream_wait(n_launched)):
            n_launched = 1
            if max_new > 1:
                launch()
            while True:
                seen = min(eng.stream_wait(n_kept + 1), n_launched)
                for row in eng.stream_read(n_kept, seen, B).to(torch.int64):
                    rows[:, n_kept] = row
                    if eos:
                        finished |= torch.isin(row, eos_t)
                    last = n_kept + 1 == max_new or (bool(eos) and bool(finished.all()))
                    if not last and n_kept >= n_launched - 2 and n_launched < max_new:
                        launch()                                          # before the callbacks: keep the device busy
                    n_kept += 1
                    if publish(row, n_kept) or last:
                        return n_kept

    # ---- sampling / EOS on the device: one fused kernel per step inside the decode graph ---------------------
    def _device_sampler_spec(self, gc, eos, pad, min_new, extra_processors, crit, processors):
        """-> a native sampler spec when this call can run entirely on the device, else None (host logits-processor path).
        On the device: greedy or sampling with repetition_penalty / no_repeat_ngram_size / temperature / top_k (1..1024) / top_p and
        up to 4 EOS ids -- the reference's DEFAULT_GENERATION_CONFIG (ref modeling_utils.py:36-47) is such a call.  Anything else
        (custom processors, stopping criteria, TFS / Top-A / Mirostat, top_k disabled, logits or scores requested) keeps the
        per-step host path; generate() streams on the device by calling this without its Stream criteria."""
        eng = self._engine
        if os.environ.get("VCLA_HOST_SAMPLER") == "1" or not hasattr(eng, "sampler_supported") or not eng.sampler_supported():
            return None
        if extra_processors or crit or getattr(gc, "output_logits", False) or getattr(gc, "output_scores", False) or len(eos) > 4:
            return None
        sampling = bool(gc.do_sample)
        rp = getattr(gc, "repetition_penalty", None) or 1.0
        ng = getattr(gc, "no_repeat_ngram_size", None) or 0
        if not sampling and rp == 1.0 and ng == 0 and not eos:
            return None                                   # plain fixed-length greedy: the argmax graphs
        if getattr(gc, "mirostat_mode", 0) == 2:
            return None
        for name, on in (("tfs", lambda v: 0.0 <= v < 1.0), ("top_a", lambda v: 0.0 < v <= 1.0), ("typical_p", lambda v: v < 1.0),
                         ("min_p", lambda v: v > 0.0), ("epsilon_cutoff", lambda v: v > 0.0), ("eta_cutoff", lambda v: v > 0.0)):
            v = getattr(gc, name, None)
            if v is not None and on(v):
                return None
        temperature = gc.temperature if (sampling and gc.temperature is not None) else 1.0
        top_k = gc.top_k if sampling else 0
        top_p = gc.top_p if (sampling and gc.top_p is not None) else 1.0
        if sampling and (top_k is None or not 1 <= top_k <= 1024 or temperature <= 0 or not 0.0 < top_p <= 1.0):
            return None
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())      # from torch's global generator: torch.manual_seed reproduces a run
        return eng.sampler_spec(do_sample=sampling, repetition_penalty=rp, no_repeat_ngram_size=ng, temperature=temperature, top_k=top_k or 0,
                                top_p=top_p, min_new_tokens=min_new, eos_token_id=eos, pad_token_id=pad, seed=seed)

    @staticmethod
    def _cut_at_eos(result, eos):
        """history rows -> the returned rows: cut where the last sequence finished (HF's per-step check); the device sampler already
        pads a finished row"""
        if not eos:
            return result
        hit = torch.zeros_like(result, dtype=torch.bool)
        for e in eos:
            hit |= result == e
        first = torch.where(hit.any(1), hit.float().argmax(1) + 1, torch.full((result.shape[0],), result.shape[1], device=result.device))
        return result[:, : int(first.max())]

    # ---- prompt lookup decoding (HF GenerationConfig.prompt_lookup_num_tokens): verification steps inside the decode graphs ----------
    LOOKUP_MAX_TOKENS = 15   # k + 1 rows fill at most the 16-column batch tile of the decode GEMMs
    LOOKUP_CHUNK = 8         # verification steps per graph replay

    LOOKUP_STREAM_CHUNK = 4  # verification steps per graph replay while streaming (two in flight: at most 8 run past a stop)

    def _lookup_tokens(self, gc, B, S, max_new) -> int:
        """-> drafted tokens per verification step of a call that runs on the device (argmax graphs, device sampler, or either of them
        streamed), or 0 when it ignores prompt_lookup_num_tokens and runs as without it: batches above one (HF refuses assisted
        generation there), VCLA_HOST_SAMPLER=1, and calls whose prompt + max_new_tokens + k exceed the context capacity.  Calls on the
        host path, beam search and generate_dp never ask."""
        k = int(getattr(gc, "prompt_lookup_num_tokens", None) or 0)
        if k < 1 or B != 1 or max_new < 2 or os.environ.get("VCLA_HOST_SAMPLER") == "1":
            return 0
        k = min(k, self.LOOKUP_MAX_TOKENS)              # speed only: the tokens are those of one-token decoding
        if S + max_new + k > self._engine.max_seq:
            return 0
        return k

    def _stream_lookup(self, start, tok, rows, max_new, eos, publish, lookup):
        """prompt lookup verification steps streamed: every wait that returns new tokens makes ONE publish of them as a (1, n) tensor
        (HF _assisted_decoding's streamer.put(valid_tokens.cpu()), then the criteria once).  Graphs of LOOKUP_STREAM_CHUNK steps are
        kept two deep: while the older one has not finished the newer one has not started, so a wait for one more token always has a
        step that will emit it until the row is final, and at most 2 x LOOKUP_STREAM_CHUNK steps run past a stop.  -> tokens kept"""
        eng = self._engine
        eos_t = torch.tensor(eos, dtype=torch.int64) if eos else None
        pending = []                                          # an event after each graph in flight
        n_kept = 0
        with self._decode_modes(start, tok, lookup, drain=lambda: [e.synchronize() for e in pending]):
            while True:
                pending = [e for e in pending if not e.query()]
                while len(pending) < 2:
                    eng.decode_many(tok, self.LOOKUP_STREAM_CHUNK)
                    pending.append(eng.record_event())
                seen = min(eng.stream_wait(n_kept + 1), max_new)
                new = eng.stream_read(n_kept, seen, 1).to(torch.int64).t()      # (1, n)
                rows[:, n_kept:seen] = new
                n_kept = seen
                # the device stops at an EOS; nothing follows it
                last = n_kept >= max_new or (bool(eos) and bool(torch.isin(new[0], eos_t).any()))
                if publish(new, n_kept) or last:
                    return n_kept

    # ---- beam search: the beam kernels and copy-on-write KV pages inside the decode graphs -------------------------------------
    def _generate_beams(self, gc, input_ids, pixel_values, attention_mask, logits_processor, stopping_criteria, streamer):
        """generate(num_beams=K, do_sample=False) with HF 5.5 semantics (HF:generation/utils.py _beam_search; the reference forwards
        num_beams to HF generate(inputs_embeds=...), ref modeling_visualcla.py:382-391).  Batches are split into chunks of
        max_batch // K prompts; each chunk runs graphs of 8 steps with one host poll of the per-item done flags between them.
        -> (B * num_return_sequences, L) int64, every row filled past its hypothesis with HF's output_fill_value."""
        K = int(gc.num_beams)
        nrs = int(getattr(gc, "num_return_sequences", 1) or 1)
        if not hasattr(self._engine, "set_beam"):
            raise NotImplementedError("this engine has no beam-search kernels")
        if gc.do_sample:
            raise NotImplementedError("beam sampling (do_sample=True with num_beams > 1) is not on the H100 path")
        if logits_processor or stopping_criteria:
            raise NotImplementedError("custom logits_processor / stopping_criteria are not supported with beam search on the H100 path")
        if streamer is not None:
            raise NotImplementedError("streaming is not supported with beam search")
        if getattr(gc, "output_scores", False) or getattr(gc, "output_logits", False):
            raise NotImplementedError("output_scores / output_logits are not supported with beam search on the H100 path")
        if (getattr(gc, "num_beam_groups", 1) or 1) > 1 or (getattr(gc, "diversity_penalty", 0.0) or 0.0) != 0.0 \
                or getattr(gc, "constraints", None) or getattr(gc, "force_words_ids", None):
            raise NotImplementedError("diverse / constrained beam search is not supported on the H100 path")
        eos = self._eos_set(gc)
        if len(eos) > 4:
            raise NotImplementedError("beam search supports at most 4 eos_token_id values")
        eng = self._engine
        if K > min(eng.max_batch, 64) or K > 16:
            raise NotImplementedError(f"num_beams={K} exceeds this model instance (at most min(max_batch, 64) rows, 16 beams)")
        max_new = gc.max_new_tokens if gc.max_new_tokens is not None else max(int(gc.max_length or 20), 1)
        es = gc.early_stopping
        spec = eng.beam_spec(K, max_new, length_penalty=gc.length_penalty if gc.length_penalty is not None else 1.0,
                             early_stopping=es if es in (True, "never") else False, eos_token_id=eos,
                             repetition_penalty=getattr(gc, "repetition_penalty", None) or 1.0,
                             no_repeat_ngram_size=getattr(gc, "no_repeat_ngram_size", None) or 0,
                             min_new_tokens=int(getattr(gc, "min_new_tokens", 0) or 0))
        pad = gc.pad_token_id if gc.pad_token_id is not None else (eos[0] if eos else None)
        fill = (pad if pad else eos[0]) if eos else -1                       # HF:3187 output_fill_value (operator precedence kept)
        chunk = max(1, min(eng.max_batch, 64) // K)
        B = input_ids.shape[0]
        toks, lens = [], []
        mode = None
        for s0 in range(0, B, chunk):
            sl = slice(s0, s0 + chunk)
            ids = input_ids[sl]
            px = None if pixel_values is None else pixel_values[sl]
            mode, rows = self._image_layout(ids, px)
            pads = self._left_pad(None if attention_mask is None else attention_mask[sl], mode)
            S = ids.shape[1] + (eng.nq if mode == N.IMAGE_AT_HEAD else 0)
            if S + max_new > eng.max_seq:
                raise ValueError(f"prompt ({S}) + max_new_tokens ({max_new}) exceeds the context capacity max_seq={eng.max_seq} "
                                 f"of this model instance")
            if mode != N.TEXT_ONLY:
                eng.vision_encode(px)
            n = ids.shape[0]
            eng.set_beam(spec)
            try:
                _, first, _ = eng.prefill(ids, mode, rows, all_logits=False, last_logits=False, left_pad=pads, pos_from_mask=True)
                tok = eng.token_buffer(n * K)
                tok.copy_(first)
                self._decode_polled(tok, max_new, lambda: eng.read_beam_done(n))
                t, ln, _, _ = eng.read_beams(n)
            finally:
                eng.set_beam(None)
            toks.append(t[:, :nrs].reshape(n * nrs, -1))
            lens.append(ln[:, :nrs].reshape(-1))
        lens = torch.cat(lens)
        L = int(lens.max())
        out = torch.full((B * nrs, L), fill, dtype=torch.int64)
        allt = torch.cat(toks).to(torch.int64)
        for i in range(B * nrs):
            out[i, : int(lens[i])] = allt[i, : int(lens[i])]
        out = out.to(eng.device)
        if not getattr(gc, "return_dict_in_generate", False):
            return out
        # the returned hypotheses need not be resident in any cache row: the handle records no ids, so it is never reused
        return SimpleNamespace(sequences=out, logits=None, scores=None,
                               past_key_values=VclaKVCache(eng, getattr(eng, "session", 0), None, mode, None))

    def _plan_kv_reuse(self, cache, input_ids, pixel_values, mode, rows, pads):
        """-> (tokens to keep, (1, T) ids to extend by) when the KV cache `cache` describes can serve this prompt, else None (full
        prefill).  Reuse needs one unpadded sequence, a current handle, the same placeholder / text-only layout and pixels, and a
        longest common prefix (LCP) of the cached and the new ids that covers the image block.  The LCP decides, not an assumption
        about tokenization: re-tokenized history often differs from the generated ids near the start of a reply."""
        eng = self._engine
        if not isinstance(cache, VclaKVCache) or cache.ids is None or not cache.is_current(eng):
            return None
        if input_ids.shape[0] != 1 or pads is not None or mode == N.IMAGE_AT_HEAD or cache.mode != mode:
            return None
        if (pixel_values is None) != (cache.pixel_values is None):
            return None
        if pixel_values is not None:
            px = pixel_values.detach().to(cache.pixel_values.device)
            if px.shape != cache.pixel_values.shape or px.dtype != cache.pixel_values.dtype or not torch.equal(px, cache.pixel_values):
                return None
        new = input_ids[0].detach().to("cpu", torch.int64)
        old = cache.ids
        n = min(new.numel(), old.numel())
        diff = torch.nonzero(new[:n] != old[:n])
        lcp = int(diff[0]) if diff.numel() else n
        keep = lcp if lcp < new.numel() else new.numel() - 1        # the whole prompt is cached: recompute its last token
        image_end = 0
        if mode == N.IMAGE_PLACEHOLDER and rows is not None and int(rows[0]) >= 0:
            image_end = int(rows[0]) + eng.nq + 1                     # <img> ... </img> stay whole
        if keep < max(image_end, 1) or new.numel() - keep > getattr(eng, "max_prefill_tokens", new.numel()):
            return None
        return keep, new[keep:].unsqueeze(0)

    @staticmethod
    def _build_processors(gc, extra):
        """HF logits processors for the sampling knobs of DEFAULT_GENERATION_CONFIG
        (ref: models/visualcla/modeling_utils.py:36-47).  Order follows HF's _get_logits_processor."""
        from transformers.generation import logits_process as lp
        procs = []
        rp = getattr(gc, "repetition_penalty", None)
        if rp is not None and rp != 1.0:
            procs.append(lp.RepetitionPenaltyLogitsProcessor(penalty=rp))
        ng = getattr(gc, "no_repeat_ngram_size", None)
        if ng is not None and ng > 0:
            procs.append(lp.NoRepeatNGramLogitsProcessor(ng))
        if extra:
            procs.extend(list(extra))
        if gc.do_sample:
            if gc.temperature is not None and gc.temperature != 1.0:
                procs.append(lp.TemperatureLogitsWarper(gc.temperature))
            if gc.top_k is not None and gc.top_k != 0:
                procs.append(lp.TopKLogitsWarper(top_k=gc.top_k, min_tokens_to_keep=1))
            if gc.top_p is not None and gc.top_p < 1.0:
                procs.append(lp.TopPLogitsWarper(top_p=gc.top_p, min_tokens_to_keep=1))
            from . import modeling_utils as mu
            if getattr(gc, "mirostat_mode", 0) == 2:
                # ref modeling_utils.py:366-371: Mirostat v2 joins the warpers and "disables samplers other than temperature" with a
                # remove-while-iterating loop -- which skips the element after every removal (temperature, top-k, top-p -> top-p
                # survives).  Replayed literally so the same generation config samples from the same distribution.
                n_fixed = len(procs) - sum(isinstance(p, (lp.TemperatureLogitsWarper, lp.TopKLogitsWarper, lp.TopPLogitsWarper)) for p in procs)
                warpers = procs[n_fixed:]
                for w in warpers:
                    if not isinstance(w, lp.TemperatureLogitsWarper):
                        warpers.remove(w)
                procs = procs[:n_fixed] + warpers
                procs.append(mu.MirostatLogitsWarper(mirostat_mode=2, mirostat_tau=getattr(gc, "mirostat_tau", 5), mirostat_eta=getattr(gc, "mirostat_eta", 0.1)))
                return procs
            for name, kw in (("tfs", "tfs"), ("top_a", "top_a")):
                val = getattr(gc, name, None)
                if val is not None and ((name == "tfs" and 0.0 <= val < 1.0) or (name == "top_a" and 0.0 < val <= 1.0)):
                    procs.append(mu.TailFreeLogitsWarper(tfs=val) if name == "tfs" else mu.TopALogitsWarper(top_a=val))
        return procs
