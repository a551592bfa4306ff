"""`visualcla` -- drop-in replacement of the reference package's public surface
(ref: models/visualcla/__init__.py:1-8), backed by hand-written sm_90a CUDA kernels (libvcla.so)."""
from .modeling_visualcla import VisualCLAModel
from .configuration_visualcla import VisualCLAConfig
from .processing_visualcla import VisualCLAProcessor
from .modeling_utils import get_model_and_tokenizer_and_processor
from .modeling_utils import chat, chat_in_stream, hijack_samplers
from .lora import load_lora

__all__ = ["VisualCLAModel", "VisualCLAConfig", "VisualCLAProcessor", "get_model_and_tokenizer_and_processor",
           "chat", "chat_in_stream", "hijack_samplers", "load_lora"]
