"""Import shim that lets the UNMODIFIED reference package (`<reference checkout>/models/visualcla`, located by
$VCLA_REFERENCE_MODELS = `<reference checkout>/models`) import and run under transformers 5.5.0.  TEST INFRASTRUCTURE ONLY
(used by oracle/gen_golden.py to produce tests/golden; no test and nothing at run time imports this).

Why each patch is needed (SURVEY.md section 8c):
  * transformers.pytorch_utils.find_pruneable_heads_and_indices   removed in 5.x
      (imported at ref: models/visualcla/modeling_visual_resampler.py:14, only used by prune_heads)
  * transformers.LogitsWarper                                     removed in 5.x
      (imported at ref: models/visualcla/modeling_utils.py:18-23)
  * PreTrainedModel.get_head_mask                                 removed in 5.x
      (called at ref: modeling_visual_resampler.py:703 with head_mask=None)
  * config.is_decoder / add_cross_attention / chunk_size_feed_forward are no longer default
      PretrainedConfig attributes -> pass them in visual_resampler_config.
"""
import os
import sys

REFERENCE_MODELS = os.environ.get("VCLA_REFERENCE_MODELS", "")


def import_reference():
    if not os.path.isdir(os.path.join(REFERENCE_MODELS, "visualcla")):
        raise RuntimeError(f"reference package not found under {REFERENCE_MODELS}")
    import transformers
    # force the lazy-module swap first, otherwise the monkey patches below are dropped
    from transformers import LlamaForCausalLM, LlamaConfig, CLIPImageProcessor, LlamaTokenizer  # noqa: F401
    import transformers.generation.logits_process as lp
    from transformers import pytorch_utils as pu
    from transformers.modeling_utils import PreTrainedModel

    def _no_prune(*a, **k):
        raise NotImplementedError("head pruning is not on the hot path")

    pu.find_pruneable_heads_and_indices = _no_prune
    lp.LogitsWarper = lp.LogitsProcessor
    sys.modules["transformers"].LogitsWarper = lp.LogitsProcessor
    transformers.LogitsWarper = lp.LogitsProcessor
    PreTrainedModel.get_head_mask = lambda self, head_mask, n_layers, *a, **k: [None] * n_layers
    if REFERENCE_MODELS not in sys.path:
        sys.path.insert(0, REFERENCE_MODELS)
    import visualcla  # the reference's package, unmodified
    assert os.path.realpath(visualcla.__file__).startswith(os.path.realpath(REFERENCE_MODELS)), \
        f"imported {visualcla.__file__}, not the reference"
    return visualcla


RESAMPLER_EXTRA = dict(is_decoder=False, add_cross_attention=False, chunk_size_feed_forward=0)
