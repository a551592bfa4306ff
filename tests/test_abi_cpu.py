"""The C-ABI library builds, loads without a GPU, and exports exactly what include/vcla.h declares.  CPU only
(no compute calls)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from visualcla import _native
    return _native.load()


def _header_symbols():
    txt = open(os.path.join(ROOT, "include", "vcla.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(vcla_[a-z0-9_]+)\s*\(", txt)))


def test_header_symbols_all_exported(lib):
    syms = _header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/vcla.h but not exported by libvcla.so"


def test_binding_covers_header():
    from visualcla import _native
    assert sorted(_native.EXPORTED_SYMBOLS) == _header_symbols()


def _header_text():
    txt = open(os.path.join(ROOT, "include", "vcla.h")).read()
    return re.sub(r"/\*.*?\*/", "", txt, flags=re.S)


def _c_kind(decl):
    decl = decl.strip()
    if "*" in decl or "[" in decl or decl.startswith("vcla_stream"):      # arrays decay to pointers
        return "ptr"
    for prefix, kind in (("float", "float"), ("int64_t", "i64"), ("uint32_t", "u32"), ("int", "int")):
        if decl.startswith(prefix):
            return kind
    raise AssertionError(f"unclassified C parameter: {decl!r}")


def _py_kind(t):
    if t is C.c_float:
        return "float"
    if t is C.c_int64:
        return "i64"
    if t is C.c_uint32:
        return "u32"
    if t is C.c_int:
        return "int"
    return "ptr"            # c_void_p / c_char_p / POINTER(...)


def test_binding_argtypes_match_prototypes():
    """Every ctypes signature has the arity and the per-argument class (pointer / int / int64 / float) of the C prototype:
    a 64-bit pointer passed as a default-int, or a float passed as an int, would corrupt the call silently."""
    from visualcla import _native
    protos = {}
    for m in re.finditer(r"[\w\s\*]+?\b(vcla_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", _header_text()):
        args = m.group(2).replace("\n", " ").strip()
        protos[m.group(1)] = [] if args in ("", "void") else [a for a in args.split(",")]
    assert sorted(protos) == _header_symbols()
    for name, _res, argtypes in _native._SIGNATURES:
        want = [_c_kind(a) for a in protos[name]]
        got = [_py_kind(t) for t in argtypes]
        assert got == want, f"{name}: header {want} vs ctypes {got}"


def test_config_struct_matches_header():
    """VclaConfig's field order and types are those of `vcla_config` in include/vcla.h."""
    from visualcla import _native
    body = re.search(r"typedef struct \{(.*?)\} vcla_config;", _header_text(), flags=re.S).group(1)
    fields = []
    for stmt in body.split(";"):
        stmt = stmt.strip()
        if not stmt:
            continue
        ctype, names = stmt.split(None, 1)
        fields += [(n.strip(), ctype) for n in names.split(",")]
    want = [(n, {"int": C.c_int, "float": C.c_float}[t]) for n, t in fields]
    assert list(_native.VclaConfig._fields_) == want
    assert C.sizeof(_native.VclaConfig) == 4 * len(want)


def test_version_and_error_strings(lib):
    assert b"sm_90a" in lib.vcla_version()
    assert isinstance(lib.vcla_last_error(), bytes)


def _tiny_config():
    from visualcla import _native
    return _native.VclaConfig(v_hidden=128, v_layers=1, v_heads=2, v_ffn=256, v_patch=14, v_image=56, v_eps=1e-5,
                              r_hidden=128, r_layers=1, r_heads=2, r_ffn=256, r_queries=8, r_eps=1e-12,
                              t_hidden=256, t_layers=1, t_heads=2, t_ffn=448, t_vocab=100, t_eps=1e-6, rope_theta=1e4,
                              max_batch=1, max_seq=32, max_prefill_tokens=32, page_tokens=16)


@pytest.mark.parametrize("var,value", [("VCLA_DECODE_SCHEDULE", "fix"), ("VCLA_DECODE_SCHEDULE", "unfused"),
                                       ("VCLA_FUSED_DECODE", "1"), ("VCLA_PREFILL_FUSED", "0")])
def test_removed_schedule_switches_refused(lib, monkeypatch, var, value):
    """A switch of a removed schedule makes vcla_create fail (before it looks for a device) and name the switch, so an old A/B
    script cannot measure the default schedule under the alternative's name."""
    monkeypatch.setenv(var, value)
    ctx = C.c_void_p()
    assert lib.vcla_create(C.byref(_tiny_config()), C.byref(ctx)) != 0
    err = lib.vcla_last_error()
    assert var.encode() in err and b"removed" in err


def test_no_cpu_fallback(lib):
    """Without a CUDA device the product must fail loudly, never compute on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    from visualcla import _native
    ctx = C.c_void_p()
    rc = lib.vcla_create(C.byref(_tiny_config()), C.byref(ctx))
    assert rc != 0 and b"no CUDA device" in lib.vcla_last_error()
    import visualcla
    with pytest.raises(_native.NativeError):
        visualcla.VisualCLAModel.from_synthetic("7b")


def test_product_never_imports_oracle():
    """Only tests/, smoke() and bench.py's CPU legs may execute oracle/ (comments may cite it)."""
    pkg = os.path.join(ROOT, "visual-chinese-llama-alpaca_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(d, f)
            if f.endswith(".py"):
                for line in open(path):
                    assert not re.match(r"\s*(import|from)\s+\S*oracle", line), (path, line)
                    assert "sys.path" not in line or "oracle" not in line, (path, line)
            elif f.endswith((".cu", ".cuh", ".h")):
                for line in open(path):
                    assert not ("#include" in line and "oracle" in line), (path, line)
    for f in os.listdir(os.path.join(ROOT, "tools")):           # the developer tools drive the product path only
        if f.endswith(".py"):
            for line in open(os.path.join(ROOT, "tools", f)):
                assert not re.match(r"\s*(import|from)\s+\S*oracle", line), (f, line)
