"""VisualCLAConfig: composite configuration (text + vision + resampler), loadable from the reference's
`config.json`.  Mirrors ref: models/visualcla/configuration_visualcla.py:10-39 (same attribute names so that
reference checkpoints load unchanged)."""
from typing import Dict, Optional, Union

from transformers.configuration_utils import PretrainedConfig


def _as_dict(cfg) -> Optional[Dict]:
    if cfg is None:
        return None
    return cfg.to_dict() if isinstance(cfg, PretrainedConfig) else dict(cfg)


class VisualCLAConfig(PretrainedConfig):
    model_type = "visualcla"
    is_composition = True

    def __init__(self, text_config: Union[PretrainedConfig, Dict, None] = None,
                 vision_config: Union[PretrainedConfig, Dict, None] = None, initializer_range: float = 0.02,
                 layer_norm_eps: float = 1e-12, use_visual_resampler: bool = False,
                 visual_resampler_config: Optional[Dict] = None, **kwargs):
        super().__init__(**kwargs)
        self.text_config = _as_dict(text_config)
        self.vision_config = _as_dict(vision_config)
        self.initializer_range = initializer_range
        self.layer_norm_eps = layer_norm_eps
        self.use_visual_resampler = use_visual_resampler
        self.visual_resampler_config = visual_resampler_config

    # ---- translation to the native path config (include/vcla.h: vcla_config) -------------------
    def to_path_config(self) -> Dict:
        t, v, r = self.text_config or {}, self.vision_config or {}, self.visual_resampler_config or {}
        if not self.use_visual_resampler:
            raise NotImplementedError("the H100 path implements the resampler variant only (VisualCLA-7B-v0.1 ships "
                                      "use_visual_resampler=True)")
        rope = t.get("rope_theta", None)
        if rope is None:
            rope = (t.get("rope_parameters") or {}).get("rope_theta", 10000.0)
        kvh = t.get("num_key_value_heads", t["num_attention_heads"])
        if kvh != t["num_attention_heads"]:
            raise NotImplementedError("grouped-query attention is not on this path (LLaMA-7B is MHA)")
        if v.get("hidden_act", "quick_gelu") != "quick_gelu":
            raise NotImplementedError("CLIP hidden_act must be quick_gelu")
        if r.get("hidden_act", "gelu") != "gelu":
            raise NotImplementedError("resampler hidden_act must be gelu")
        return dict(
            v_hidden=v["hidden_size"], v_layers=v["num_hidden_layers"], v_heads=v["num_attention_heads"],
            v_ffn=v["intermediate_size"], v_patch=v["patch_size"], v_image=v["image_size"],
            v_eps=v.get("layer_norm_eps", 1e-5),
            r_hidden=r.get("hidden_size", 768), r_layers=r.get("num_hidden_layers", 12),
            r_heads=r.get("num_attention_heads", 12), r_ffn=r.get("intermediate_size", 3072),
            r_queries=r.get("num_query_tokens", 32), r_eps=r.get("layer_norm_eps", 1e-12),
            t_hidden=t["hidden_size"], t_layers=t["num_hidden_layers"], t_heads=t["num_attention_heads"],
            t_ffn=t["intermediate_size"], t_vocab=t["vocab_size"], t_eps=t.get("rms_norm_eps", 1e-6),
            rope_theta=float(rope))

    @classmethod
    def from_path_config(cls, p: Dict) -> "VisualCLAConfig":
        text = dict(model_type="llama", vocab_size=p["t_vocab"], hidden_size=p["t_hidden"], intermediate_size=p["t_ffn"],
                    num_hidden_layers=p["t_layers"], num_attention_heads=p["t_heads"], num_key_value_heads=p["t_heads"],
                    rms_norm_eps=p["t_eps"], rope_theta=p["rope_theta"], max_position_embeddings=2048,
                    hidden_act="silu", tie_word_embeddings=False, bos_token_id=1, eos_token_id=2, pad_token_id=0)
        vision = dict(model_type="clip_vision_model", hidden_size=p["v_hidden"], intermediate_size=p["v_ffn"],
                      num_hidden_layers=p["v_layers"], num_attention_heads=p["v_heads"], image_size=p["v_image"],
                      patch_size=p["v_patch"], hidden_act="quick_gelu", layer_norm_eps=p["v_eps"], num_channels=3)
        res = dict(hidden_size=p["r_hidden"], num_hidden_layers=p["r_layers"], num_attention_heads=p["r_heads"],
                   intermediate_size=p["r_ffn"], hidden_act="gelu", layer_norm_eps=p["r_eps"],
                   num_query_tokens=p["r_queries"])
        return cls(text_config=text, vision_config=vision, use_visual_resampler=True, visual_resampler_config=res)
