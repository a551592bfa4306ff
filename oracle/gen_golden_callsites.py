"""Extract the call sites tests/test_dropin_conformance_cpu.py checks from the unmodified reference into
tests/golden/reference_call_sites.json (data only: attribute chains, keyword names, positional counts, imported names and
the loader's parameter names).  Run once with the reference tree available:

    python oracle/gen_golden_callsites.py /path/to/Visual-Chinese-LLaMA-Alpaca
"""
import ast
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = ["inference.py", "gradio_demo.py"]
LOADER_FNS = ["get_model_and_tokenizer_and_processor", "chat", "chat_in_stream", "encoding_text"]


def calls(tree, root_name):
    """(attribute chain, keyword names, n positional) of every call whose function is an attribute chain starting at `root_name`."""
    out = []
    for node in ast.walk(tree):
        if not isinstance(node, ast.Call):
            continue
        chain, f = [], node.func
        while isinstance(f, ast.Attribute):
            chain.append(f.attr)
            f = f.value
        if isinstance(f, ast.Call):          # e.g. model.text_model.get_input_embeddings().weight.size(0): follow the inner call too
            continue
        if isinstance(f, ast.Name) and f.id == root_name and chain:
            out.append([list(reversed(chain)), [k.arg for k in node.keywords if k.arg], len(node.args)])
    return out


def main(ref):
    data = {"scripts": {}, "loader_params": {}}
    for script in SCRIPTS:
        tree = ast.parse(open(os.path.join(ref, "scripts", "inference", script)).read())
        imports = [[n.module, [a.name for a in n.names]] for n in ast.walk(tree)
                   if isinstance(n, ast.ImportFrom) and n.module and n.module.startswith("visualcla")]
        data["scripts"][script] = {"visualcla_calls": calls(tree, "visualcla"), "imports": imports,
                                   "model_calls": {r: calls(tree, r) for r in ("model", "base_model")}}
    tree = ast.parse(open(os.path.join(ref, "models", "visualcla", "modeling_utils.py")).read())
    defs = {n.name: n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef)}
    for fn in LOADER_FNS:
        data["loader_params"][fn] = [a.arg for a in defs[fn].args.args]
    out = os.path.join(ROOT, "tests", "golden", "reference_call_sites.json")
    with open(out, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)
        f.write("\n")
    print(out)


if __name__ == "__main__":
    main(sys.argv[1])
