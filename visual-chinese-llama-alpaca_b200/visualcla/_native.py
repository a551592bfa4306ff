"""ctypes binding of libvcla.so (include/vcla.h).  No CPU fallback: if the library or a CUDA
device is missing every entry point raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libvcla.so")

VCLA_F32, VCLA_F16, VCLA_BF16 = 0, 1, 2
TEXT_ONLY, IMAGE_AT_HEAD, IMAGE_PLACEHOLDER = 0, 1, 2


class VclaConfig(C.Structure):
    _fields_ = [
        ("v_hidden", C.c_int), ("v_layers", C.c_int), ("v_heads", C.c_int), ("v_ffn", C.c_int),
        ("v_patch", C.c_int), ("v_image", C.c_int), ("v_eps", C.c_float),
        ("r_hidden", C.c_int), ("r_layers", C.c_int), ("r_heads", C.c_int), ("r_ffn", C.c_int),
        ("r_queries", C.c_int), ("r_eps", C.c_float),
        ("t_hidden", C.c_int), ("t_layers", C.c_int), ("t_heads", C.c_int), ("t_ffn", C.c_int),
        ("t_vocab", C.c_int), ("t_eps", C.c_float), ("rope_theta", C.c_float),
        ("max_batch", C.c_int), ("max_seq", C.c_int), ("max_prefill_tokens", C.c_int), ("page_tokens", C.c_int),
        ("weight_format", C.c_int), ("kv_format", C.c_int),
    ]


class VclaSampler(C.Structure):
    _fields_ = [("do_sample", C.c_int), ("repetition_penalty", C.c_float), ("no_repeat_ngram_size", C.c_int), ("temperature", C.c_float),
                ("top_k", C.c_int), ("top_p", C.c_float), ("min_new_tokens", C.c_int), ("n_eos", C.c_int), ("eos_token_id", C.c_int * 4),
                ("pad_token_id", C.c_int), ("seed", C.c_uint64)]


class VclaBeam(C.Structure):
    _fields_ = [("num_beams", C.c_int), ("length_penalty", C.c_float), ("early_stopping", C.c_int), ("max_new_tokens", C.c_int),
                ("n_eos", C.c_int), ("eos_token_id", C.c_int * 4), ("repetition_penalty", C.c_float), ("no_repeat_ngram_size", C.c_int),
                ("min_new_tokens", C.c_int)]


class VclaLookup(C.Structure):
    _fields_ = [("k", C.c_int), ("n", C.c_int), ("max_new", C.c_int), ("prompt_ids", C.c_void_p), ("prompt_len", C.c_int)]


class NativeError(RuntimeError):
    pass


_lib = None

# every symbol include/vcla.h declares: (name, restype, argtypes)
_P = C.c_void_p
_SIGNATURES = [
    ("vcla_last_error", C.c_char_p, []),
    ("vcla_version", C.c_char_p, []),
    ("vcla_create", C.c_int, [C.POINTER(VclaConfig), C.POINTER(_P)]),
    ("vcla_destroy", None, [_P]),
    ("vcla_get_config", C.c_int, [_P, C.POINTER(VclaConfig)]),
    ("vcla_memory_bytes", C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("vcla_weight_count", C.c_int, [_P]),
    ("vcla_weight_info", C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64 * 4), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("vcla_load_weight", C.c_int, [_P, C.c_char_p, _P, C.c_int, C.c_int64, C.c_int, _P]),
    ("vcla_read_weight", C.c_int, [_P, C.c_char_p, _P, _P]),
    ("vcla_init_synthetic", C.c_int, [_P, C.c_uint32, _P]),
    ("vcla_read_weight_q8", C.c_int, [_P, C.c_char_p, _P, _P, _P]),
    ("vcla_load_weight_q8", C.c_int, [_P, C.c_char_p, _P, _P, C.c_int, _P]),
    ("vcla_reset", C.c_int, [_P, _P]),
    ("vcla_kv_geometry", C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("vcla_kv_read_layer", C.c_int, [_P, C.c_int, _P]),
    ("vcla_kv_read_pages", C.c_int, [_P, _P, _P, _P]),
    ("vcla_kv_debug_shuffle", C.c_int, [_P, C.c_uint32]),
    ("vcla_kv_truncate", C.c_int, [_P, _P, C.c_int, _P]),
    ("vcla_vision_encode", C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    ("vcla_prefill", C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P]),
    ("vcla_prefill_extend", C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, _P, _P]),
    ("vcla_decode_step", C.c_int, [_P, _P, C.c_int, _P, _P, C.c_int, _P]),
    ("vcla_decode_multi", C.c_int, [_P, _P, C.c_int, C.c_int, _P]),
    ("vcla_read_history", C.c_int, [_P, _P, C.c_int, C.c_int, _P]),
    ("vcla_sampler_supported", C.c_int, [_P]),
    ("vcla_set_sampler", C.c_int, [_P, C.POINTER(VclaSampler), _P]),
    ("vcla_read_finished", C.c_int, [_P, _P, C.c_int, _P]),
    ("vcla_op_sample", C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, C.POINTER(VclaSampler), _P, _P, _P]),
    # prompt lookup decoding (HF:generation/candidate_generator.py PromptLookupCandidateGenerator, HF:generation/utils.py _assisted_decoding)
    ("vcla_set_lookup", C.c_int, [_P, C.POINTER(VclaLookup), _P]),
    ("vcla_read_lookup_stats", C.c_int, [_P, _P, _P]),
    ("vcla_set_beam", C.c_int, [_P, C.POINTER(VclaBeam)]),
    ("vcla_set_fanout", C.c_int, [_P, C.c_int]),
    ("vcla_read_beams", C.c_int, [_P, _P, _P, _P, _P]),
    ("vcla_beam_cow_bytes", C.c_int, [_P, C.POINTER(C.c_int64), C.c_int]),
    ("vcla_op_beam_step", C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, C.POINTER(VclaBeam), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    ("vcla_nccl_unique_id", C.c_int, [_P]),
    ("vcla_nccl_init", C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int]),
    ("vcla_allgather_tokens", C.c_int, [_P, _P, C.c_int, _P, _P]),
    ("vcla_dp_set_active", C.c_int, [_P, C.c_int]),
    ("vcla_dp_exchange", C.c_int, [_P, _P]),
    ("vcla_read_history_dp", C.c_int, [_P, _P, C.c_int, _P]),
    # token streaming (ref: models/visualcla/modeling_utils.py:180-247 chat_in_stream; HF generate(streamer=...))
    ("vcla_stream_arm", C.c_int, [_P, C.c_int]),
    ("vcla_stream_wait", C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    ("vcla_stream_read", C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    ("vcla_kernel_launches", C.c_int64, [_P, C.c_int]),
    ("vcla_read_stage", C.c_int, [_P, C.c_char_p, C.c_int, _P, _P]),
    ("vcla_op_gemm", C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    ("vcla_op_gemm_csk", C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, _P]),
    ("vcla_op_gemm_csk_clusters", C.c_int, [C.c_int, C.c_int]),
    ("vcla_op_gemm_csk_q8", C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, _P]),
    ("vcla_op_gemm_q8", C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P, _P]),
    ("vcla_debug_set_csk_splits", C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    ("vcla_debug_get_csk_splits", C.c_int, [_P, C.c_int, C.POINTER(C.c_int * 5)]),
    ("vcla_debug_decode_ctas_per_sm", C.c_int, [_P, C.c_int, C.POINTER(C.c_int * 2)]),
    ("vcla_set_attention_tc", None, [C.c_int]),
    ("vcla_op_attention", C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, _P, C.c_int,
                                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _P, _P]),
    ("vcla_op_attention_paged", C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_float, _P]),
    ("vcla_op_attention_decode", C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float,
                                           C.c_float, C.c_int, C.c_int, C.c_int, _P]),
    ("vcla_op_attention_decode_lookup", C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float,
                                                  C.c_float, _P]),
    ("vcla_op_attention_paged_q8", C.c_int, [_P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_float, _P]),
    ("vcla_op_attention_decode_q8", C.c_int, [_P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float,
                                              C.c_float, C.c_int, C.c_int, C.c_int, _P]),
    ("vcla_op_attention_decode_lookup_q8", C.c_int, [_P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int,
                                                     C.c_float, C.c_float, _P]),
    ("vcla_op_logits_argmax", C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    ("vcla_op_layernorm", C.c_int, [_P, C.c_int, C.c_int, _P, _P, C.c_float, _P, _P, _P]),
    ("vcla_op_rmsnorm", C.c_int, [_P, C.c_int, C.c_int, _P, C.c_float, _P, _P]),
    ("vcla_bench_decode_gemm", C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int64), _P]),
    ("vcla_trace_enable", C.c_int, [_P, C.c_int]),
    ("vcla_trace_read", C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_int)]),
    ("vcla_set_pdl", None, [C.c_int]),
    ("vcla_preprocess_workspace_bytes", C.c_int64, [C.c_int, C.c_int, C.c_int]),
    ("vcla_resample_taps", C.c_int, [C.c_int, C.c_int, _P, _P, _P, C.c_int]),
    ("vcla_preprocess_image", C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, C.c_int64, _P,
                                        C.c_int, _P]),
]
EXPORTED_SYMBOLS = [s[0] for s in _SIGNATURES]


def load():
    """Load libvcla.so (once).  Raises NativeError if it was not built -- there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(f"{LIB_PATH} not found: build it with `python visual-chinese-llama-alpaca_b200/build.py` "
                          "(or __graft_entry__.build()); this package has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    for name, res, args in _SIGNATURES:
        fn = getattr(lib, name)          # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    if os.environ.get("VCLA_PDL", "") not in ("", "0"):
        lib.vcla_set_pdl(1)        # programmatic dependent launch for every kernel enqueued afterwards
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().vcla_last_error()
        raise NativeError(f"{what}: {msg.decode() if msg else 'unknown error'}")


def ptr(t):
    """device/host pointer of a torch tensor (or None)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())
