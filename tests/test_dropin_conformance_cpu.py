"""Static drop-in check against the reference's OWN call sites, pinned in tests/golden/reference_call_sites.json (extracted from the
unmodified reference by oracle/gen_golden_callsites.py; tests/test_loader_gpu.py replays the same call sequence on the device).  Every
`visualcla.<name>(...)` call in scripts/inference/inference.py and scripts/inference/gradio_demo.py must resolve in this package with a
signature that accepts the keywords the script passes, and every method / attribute the scripts touch on the model object must exist
on VisualCLAModel."""
import inspect
import json
import os

import pytest

import visualcla
from visualcla.modeling_visualcla import VisualCLAModel, _SubModel

SCRIPTS = ["inference.py", "gradio_demo.py"]


@pytest.fixture(scope="module")
def call_sites(golden_dir):
    with open(os.path.join(golden_dir, "reference_call_sites.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("script", SCRIPTS)
def test_reference_scripts_resolve_against_this_package(script, call_sites):
    sites = call_sites["scripts"][script]
    seen = []
    for chain, kws, npos in sites["visualcla_calls"]:
        obj = visualcla
        for name in chain:
            assert hasattr(obj, name), f"{script}: visualcla.{'.'.join(chain)} does not exist in the drop-in package"
            obj = getattr(obj, name)
        if callable(obj):
            params = inspect.signature(obj).parameters
            accepts_kwargs = any(p.kind is inspect.Parameter.VAR_KEYWORD for p in params.values())
            for k in kws:
                assert k in params or accepts_kwargs, f"{script}: visualcla.{'.'.join(chain)}() is called with {k}= which the drop-in does not accept"
            assert npos <= len([p for p in params.values() if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)])
        seen.append(".".join(chain))
    assert seen, f"{script} makes no visualcla.* call?"
    # attribute imports:  from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG  (gradio_demo.py:2)
    for module, names in sites["imports"]:
        mod = __import__(module, fromlist=["x"])
        for name in names:
            assert hasattr(mod, name), f"{script}: from {module} import {name}"
    # methods / attributes the scripts use on the model objects
    for root in ("model", "base_model"):
        for chain, _kws, _n in sites["model_calls"][root]:
            cls = VisualCLAModel
            for i, name in enumerate(chain):
                if name in ("text_model", "vision_model", "visual_resampler"):      # set per instance in __init__: handles of type _SubModel
                    cls = _SubModel
                    continue
                assert hasattr(cls, name) or name in ("tokenizer", "image_processor", "num_patch", "device", "config"), \
                    f"{script}: {root}.{'.'.join(chain)}: '{name}' is missing on {cls.__name__}"
                break
    if script == "inference.py":
        assert "get_model_and_tokenizer_and_processor" in seen and "chat" in seen


def test_loader_signature_matches_the_reference_definition(call_sites):
    """Same parameter names, order and defaults as ref models/visualcla/modeling_utils.py:83-92 (plus **engine_kwargs)."""
    for fn, want in call_sites["loader_params"].items():
        have = [p.name for p in inspect.signature(getattr(visualcla.modeling_utils, fn)).parameters.values()
                if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
        assert have[: len(want)] == want, f"{fn}: reference parameters {want}, drop-in {have}"
