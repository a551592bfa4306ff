"""Thin Python owner of a native `vcla_ctx` (include/vcla.h): creation from a path config, weight loading by
reference state-dict names, and the three phases of the path.  All tensors are torch CUDA tensors used as raw
device buffers; every kernel is enqueued on torch's current stream."""
import ctypes as C
from typing import Dict, Iterable, Optional, Tuple

import torch

from . import _native as N

_DTYPE = {torch.float32: N.VCLA_F32, torch.float16: N.VCLA_F16, torch.bfloat16: N.VCLA_BF16}

PATH_KEYS = ["v_hidden", "v_layers", "v_heads", "v_ffn", "v_patch", "v_image", "v_eps",
             "r_hidden", "r_layers", "r_heads", "r_ffn", "r_queries", "r_eps",
             "t_hidden", "t_layers", "t_heads", "t_ffn", "t_vocab", "t_eps", "rope_theta"]


def path_config_7b() -> Dict:
    """VisualCLA-7B-v0.1 shapes (SURVEY.md section 8 constants)."""
    return dict(v_hidden=1024, v_layers=24, v_heads=16, v_ffn=4096, v_patch=14, v_image=224, v_eps=1e-5,
                r_hidden=1024, r_layers=6, r_heads=16, r_ffn=4096, r_queries=64, r_eps=1e-12,
                t_hidden=4096, t_layers=32, t_heads=32, t_ffn=11008, t_vocab=49958, t_eps=1e-6, rope_theta=10000.0)


def kv_format_of(kv_cache_dtype) -> int:
    """kv_cache_dtype of the model constructors -> Engine kv_format: "int8" / torch.int8 select the int8 KV cache; None, "bfloat16"
    and torch.bfloat16 the bf16 one.  The cache format is fixed when the engine is built."""
    if kv_cache_dtype is None or kv_cache_dtype in ("bfloat16", torch.bfloat16):
        return Engine.KV_BF16
    if kv_cache_dtype in ("int8", torch.int8):
        return Engine.KV_INT8
    raise ValueError(f"kv_cache_dtype must be None, 'bfloat16', torch.bfloat16, 'int8' or torch.int8 (got {kv_cache_dtype!r})")


class Engine:
    WEIGHT_BF16, WEIGHT_INT8 = 0, 1      # weight_format: storage of the LLaMA projections (int8 = load_in_8bit, include/vcla.h)
    KV_BF16, KV_INT8 = 0, 1              # kv_format: storage of the paged KV cache (int8 = kv_cache_dtype="int8", include/vcla.h)

    def __init__(self, path_cfg: Dict, max_batch: int = 8, max_seq: int = 512, max_prefill_tokens: Optional[int] = None,
                 device: Optional[torch.device] = None, page_tokens: int = 64, weight_format: int = 0, kv_format: int = 0):
        if not torch.cuda.is_available():
            raise N.NativeError("visualcla (H100) needs a CUDA device: there is no CPU fallback")
        self.lib = N.load()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.path_cfg = {k: path_cfg[k] for k in PATH_KEYS}
        self.max_batch, self.max_seq = int(max_batch), int(max_seq)
        self.max_prefill_tokens = int(max_prefill_tokens or max_batch * max_seq)
        cfg = N.VclaConfig(**self.path_cfg, max_batch=self.max_batch, max_seq=self.max_seq,
                           max_prefill_tokens=self.max_prefill_tokens, page_tokens=page_tokens, weight_format=int(weight_format),
                           kv_format=int(kv_format))
        self.weight_format = int(weight_format)
        self.kv_format = int(kv_format)
        self._ctx = C.c_void_p()
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_create(C.byref(cfg), C.byref(self._ctx)), "vcla_create")
        self.nq = self.path_cfg["r_queries"]
        self.vocab = self.path_cfg["t_vocab"]
        self._names = None
        self._table_cache = None
        self._dp_tok = {}
        # bumped by every call that changes the cached sequences or the weights: a KV-cache handle (VclaKVCache) taken at one value
        # describes the cache only while the counter still has it
        self.session = 0

    # ---- lifetime ---------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self.lib.vcla_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def memory_bytes(self) -> Tuple[int, int, int]:
        w, k, a = C.c_int64(), C.c_int64(), C.c_int64()
        N.check(self.lib.vcla_memory_bytes(self._ctx, C.byref(w), C.byref(k), C.byref(a)), "vcla_memory_bytes")
        return w.value, k.value, a.value

    # ---- weights ----------------------------------------------------------------------------
    def weight_table(self):
        """[(name, shape, kind)] in the reference's state-dict naming; kind 0 = bf16 matrix, 1 = f32 vector, 2 = int8 matrix + row scales."""
        if self._names is None:
            out = []
            for i in range(self.lib.vcla_weight_count(self._ctx)):
                name, shape, nd, kind = C.c_char_p(), (C.c_int64 * 4)(), C.c_int(), C.c_int()
                N.check(self.lib.vcla_weight_info(self._ctx, i, C.byref(name), C.byref(shape), C.byref(nd), C.byref(kind)), "vcla_weight_info")
                out.append((name.value.decode(), tuple(shape[j] for j in range(nd.value)), kind.value))
            self._names = out
        return self._names

    def _table(self):
        if getattr(self, "_table_cache", None) is None:
            self._table_cache = {n: (s, k) for n, s, k in self.weight_table()}
        return self._table_cache

    def load_weight(self, name: str, tensor: torch.Tensor):
        """Copy one tensor (named as in the reference's state dict) into the arena.  The shape must be the slot's shape:
        a checkpoint that disagrees with config.json is an error here, never an out-of-bounds read on the native side
        (which checks the element count again)."""
        table = self._table()
        if name not in table:
            raise KeyError(f"unknown tensor '{name}' for this model configuration")
        t = tensor.detach()
        if tuple(t.shape) != tuple(table[name][0]):
            raise ValueError(f"shape mismatch for {name}: checkpoint {tuple(t.shape)} vs model {tuple(table[name][0])}")
        if t.dtype not in _DTYPE:
            t = t.float()
        t = t.contiguous()
        on_dev = 1 if t.is_cuda else 0
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_load_weight(self._ctx, name.encode(), N.ptr(t), _DTYPE[t.dtype], t.numel(), on_dev, self._stream()),
                    f"vcla_load_weight({name})")

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True, prefix: str = ""):
        table = {n: (s, k) for n, s, k in self.weight_table()}
        loaded, unexpected = set(), []
        for k, v in sd.items():
            name = prefix + k
            if name not in table:
                unexpected.append(name)
                continue
            if tuple(v.shape) != tuple(table[name][0]):
                raise ValueError(f"shape mismatch for {name}: checkpoint {tuple(v.shape)} vs model {tuple(table[name][0])}")
            self.load_weight(name, v)
            loaded.add(name)
        return loaded, unexpected

    def read_weight(self, name: str) -> torch.Tensor:
        """Host copy of one logical tensor: bf16 for kind 0, fp32 for kind 1 and for kind 2 (the int8 rows dequantised, q * s)."""
        shape, kind = self._table()[name]
        out = torch.empty(shape, dtype=torch.bfloat16 if kind == 0 else torch.float32)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_weight(self._ctx, name.encode(), N.ptr(out), self._stream()), f"vcla_read_weight({name})")
        return out

    def read_weight_q8(self, name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (q int8 (rows, cols), scale f32 (rows,)) host tensors of an int8 tensor (kind 2), exactly as stored."""
        shape, _kind = self._table()[name]
        q = torch.empty(shape, dtype=torch.int8)
        s = torch.empty(shape[0], dtype=torch.float32)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_weight_q8(self._ctx, name.encode(), N.ptr(q), N.ptr(s), self._stream()), f"vcla_read_weight_q8({name})")
        return q, s

    def load_weight_q8(self, name: str, q: torch.Tensor, scale: torch.Tensor):
        """Store int8 rows + fp32 row scales of an int8 tensor (kind 2) exactly (no requantisation)."""
        shape, _kind = self._table()[name]
        if tuple(q.shape) != tuple(shape) or q.dtype != torch.int8 or tuple(scale.shape) != (shape[0],):
            raise ValueError(f"{name}: expected int8 {tuple(shape)} and scales ({shape[0]},), got {q.dtype} {tuple(q.shape)} / {tuple(scale.shape)}")
        q = q.detach().contiguous()
        s = scale.detach().to(q.device, torch.float32).contiguous()
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_load_weight_q8(self._ctx, name.encode(), N.ptr(q), N.ptr(s), 1 if q.is_cuda else 0, self._stream()),
                    f"vcla_load_weight_q8({name})")

    def init_synthetic(self, seed: int = 0):
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_init_synthetic(self._ctx, seed, self._stream()), "vcla_init_synthetic")

    # ---- the path ---------------------------------------------------------------------------
    def vision_encode(self, pixel_values: torch.Tensor, return_embeds: bool = False) -> Optional[torch.Tensor]:
        px = pixel_values
        if px.device != self.device:
            px = px.to(self.device, non_blocking=True)
        if px.dtype not in _DTYPE:
            px = px.float()
        px = px.contiguous()
        B = px.shape[0]
        I = self.path_cfg["v_image"]
        if tuple(px.shape[1:]) != (3, I, I):
            raise ValueError(f"Input image size ({px.shape[2]}*{px.shape[3]}) doesn't match model ({I}*{I}).")
        out = torch.empty(B, self.nq, self.path_cfg["t_hidden"], dtype=torch.float32, device=self.device) if return_embeds else None
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_vision_encode(self._ctx, N.ptr(px), _DTYPE[px.dtype], B, N.ptr(out), self._stream()), "vcla_vision_encode")
        return out

    def prefill(self, input_ids: torch.Tensor, image_mode: int, img_rows: Optional[torch.Tensor] = None,
                all_logits: bool = False, last_logits: bool = True, left_pad: Optional[torch.Tensor] = None, pos_from_mask: bool = True):
        ids = input_ids.to(self.device, dtype=torch.int64).contiguous()
        B, T = ids.shape
        S = T + self.nq if image_mode == N.IMAGE_AT_HEAD else T
        la = torch.empty(B, S, self.vocab, dtype=torch.float32, device=self.device) if all_logits else None
        ll = torch.empty(B, self.vocab, dtype=torch.float32, device=self.device) if last_logits else None
        tok = torch.empty(B * (self._beam.num_beams if self._beam is not None else self._fanout), dtype=torch.int32, device=self.device)
        rows = None if img_rows is None else img_rows.to(self.device, dtype=torch.int32).contiguous()
        pad = None if left_pad is None else left_pad.to(self.device, dtype=torch.int32).contiguous()
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_prefill(self._ctx, N.ptr(ids), B, T, image_mode, N.ptr(rows), N.ptr(pad), 1 if pos_from_mask else 0,
                                          N.ptr(la), N.ptr(ll), N.ptr(tok), self._stream()), "vcla_prefill")
        return ll, tok, la

    def extend(self, input_ids: torch.Tensor, all_logits: bool = False, last_logits: bool = True):
        """Append the (B, T) tokens to the B sequences resident since the last prefill (vcla_prefill_extend): they attend to the
        cached prefix, no vision work runs.  -> (last logits (B,V) or None, picked tokens (B,) int32, logits (B,T,V) or None)."""
        ids = input_ids.to(self.device, dtype=torch.int64).contiguous()
        B, T = ids.shape
        la = torch.empty(B, T, self.vocab, dtype=torch.float32, device=self.device) if all_logits else None
        ll = torch.empty(B, self.vocab, dtype=torch.float32, device=self.device) if last_logits else None
        tok = torch.empty(B, dtype=torch.int32, device=self.device)
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_prefill_extend(self._ctx, N.ptr(ids), B, T, N.ptr(la), N.ptr(ll), N.ptr(tok), self._stream()),
                    "vcla_prefill_extend")
        return ll, tok, la

    def truncate(self, lengths):
        """Keep the first min(current, lengths[b]) cached tokens of each resident sequence (vcla_kv_truncate)."""
        n = torch.as_tensor(lengths, dtype=torch.int32).reshape(-1).contiguous()
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_kv_truncate(self._ctx, N.ptr(n), n.numel(), self._stream()), "vcla_kv_truncate")

    def decode_step(self, tok_in: torch.Tensor, tok_out: torch.Tensor, logits: Optional[torch.Tensor] = None, use_graph: bool = True):
        """tok_in / tok_out: int32 CUDA tensors of shape (B,) that stay alive (and at the same address) across steps."""
        B = tok_in.shape[0]
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_decode_step(self._ctx, N.ptr(tok_in), B, N.ptr(logits), N.ptr(tok_out), 1 if use_graph else 0,
                                              self._stream()), "vcla_decode_step")

    GRAPH_CHUNK = 16     # decode steps per CUDA graph in the fixed-length greedy loop

    def decode_many(self, tok: torch.Tensor, n_steps: int):
        """n_steps greedy steps on the in-place int32 token buffer `tok` (B,), replayed in graphs of GRAPH_CHUNK steps."""
        B = tok.shape[0]
        left = n_steps
        self.session += 1
        with torch.cuda.device(self.device):
            while left > 0:
                k = self.GRAPH_CHUNK
                while k > left:
                    k >>= 1                       # power-of-two tails: at most log2(GRAPH_CHUNK)+1 graph variants
                N.check(self.lib.vcla_decode_multi(self._ctx, N.ptr(tok), B, k, self._stream()), "vcla_decode_multi")
                left -= k

    def token_buffer(self, n: int) -> torch.Tensor:
        """Persistent int32 (n,) device buffer per batch size: its address keys the captured decode graphs."""
        if n not in self._dp_tok:
            with torch.inference_mode(False):
                self._dp_tok[n] = torch.zeros(n, dtype=torch.int32, device=self.device)
        return self._dp_tok[n]

    # ---- data parallel: communicator + in-graph token exchange (include/vcla.h, "data parallel") -------------
    dp_width = 0

    def dp_init(self, group=None):
        """Create this context's NCCL communicator once (collective over the process group): rank 0's ncclUniqueId is
        shipped through torch.distributed, the communicator itself belongs to the native context."""
        import torch.distributed as dist
        if self.dp_width:
            return
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        uid = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            N.check(self.lib.vcla_nccl_unique_id(N.ptr(uid)), "vcla_nccl_unique_id")
        uid_d = uid.to(self.device)
        src = dist.get_global_rank(group, 0) if group is not None else 0
        dist.broadcast(uid_d, src=src, group=group)
        uid = uid_d.cpu()
        width = min(64, self.max_batch)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_nccl_init(self._ctx, N.ptr(uid), rank, world, width), "vcla_nccl_init")
        self.dp_width, self.dp_world = width, world

    def dp_set_active(self, on: bool):
        N.check(self.lib.vcla_dp_set_active(self._ctx, 1 if on else 0), "vcla_dp_set_active")

    def dp_idle_exchange(self):
        """A rank that holds no requests (global batch < world) still has to enter every step's all-gather."""
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_dp_exchange(self._ctx, self._stream()), "vcla_dp_exchange")

    def allgather_tokens(self, local: torch.Tensor) -> torch.Tensor:
        out = torch.empty(self.dp_world * local.numel(), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_allgather_tokens(self._ctx, N.ptr(local), local.numel(), N.ptr(out), self._stream()), "vcla_allgather_tokens")
        return out

    def read_history_dp(self, n_steps: int) -> torch.Tensor:
        """(n_steps, world * dp_width) int32 CUDA tensor: every rank's tokens of the prefill (row 0) and each decode step."""
        out = torch.empty(n_steps, self.dp_world * self.dp_width, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_history_dp(self._ctx, N.ptr(out), n_steps, self._stream()), "vcla_read_history_dp")
        return out

    # ---- device-side sampling (include/vcla.h, "device-side sampling") -------------------------------------
    def sampler_supported(self) -> bool:
        return bool(self.lib.vcla_sampler_supported(self._ctx))

    @staticmethod
    def sampler_spec(do_sample=False, repetition_penalty=1.0, no_repeat_ngram_size=0, temperature=1.0, top_k=0, top_p=1.0,
                     min_new_tokens=0, eos_token_id=(), pad_token_id=0, seed=0) -> "N.VclaSampler":
        eos = list(eos_token_id)
        arr = (C.c_int * 4)(*(eos + [0] * (4 - len(eos)))[:4])
        return N.VclaSampler(1 if do_sample else 0, float(repetition_penalty), int(no_repeat_ngram_size or 0), float(temperature), int(top_k or 0),
                             float(top_p), int(min_new_tokens or 0), len(eos), arr, int(pad_token_id), int(seed) & (2 ** 64 - 1))

    def set_sampler(self, spec: Optional["N.VclaSampler"]):
        """spec = sampler_spec(...): prefill / decode pick tokens with the fused device sampler; None: back to argmax."""
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_set_sampler(self._ctx, C.byref(spec) if spec is not None else None, self._stream()), "vcla_set_sampler")

    def set_lookup(self, prompt_ids: Optional[torch.Tensor], k: int = 0, n: int = 2, max_new: int = 0):
        """Prompt lookup decoding of the one resident sequence (include/vcla.h): decode_many then runs verification steps of up to k
        drafts copied from prompt_ids ++ the emitted tokens (n-grams of up to n tokens).  None: plain decode steps."""
        with torch.cuda.device(self.device):
            if prompt_ids is None:
                N.check(self.lib.vcla_set_lookup(self._ctx, None, self._stream()), "vcla_set_lookup")
                return
            ids = prompt_ids.reshape(-1).to(self.device, torch.int64).contiguous()
            spec = N.VclaLookup(k=int(k), n=int(n), max_new=int(max_new), prompt_ids=ids.data_ptr(), prompt_len=ids.numel())
            N.check(self.lib.vcla_set_lookup(self._ctx, C.byref(spec), self._stream()), "vcla_set_lookup")

    def lookup_stats(self) -> Tuple[int, bool, int, int, int, int]:
        """-> (history rows, finished, verification steps that emitted, drafts offered, drafts emitted, rows per step).  Synchronises."""
        out = (C.c_int64 * 6)()
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_lookup_stats(self._ctx, out, self._stream()), "vcla_read_lookup_stats")
        return int(out[0]), bool(out[1]), int(out[2]), int(out[3]), int(out[4]), int(out[5])

    def record_event(self):
        """A CUDA event recorded on this engine's stream after the work enqueued so far (.query() is True once it has run)."""
        e = torch.cuda.Event()
        e.record(torch.cuda.current_stream(self.device))
        return e

    def read_finished(self, B: int) -> torch.Tensor:
        out = torch.empty(B, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_finished(self._ctx, N.ptr(out), B, self._stream()), "vcla_read_finished")
        return out

    def op_sample(self, logits: torch.Tensor, history: Optional[torch.Tensor], spec: "N.VclaSampler", return_scores: bool = True):
        """The sampler kernel on caller data: logits (B,V) f32, history (B,L) tokens.  -> (tokens (B,) int32, processed scores (B,V))."""
        lg = logits.to(self.device, torch.float32).contiguous()
        B, V = lg.shape
        L = 0 if history is None else history.shape[1]
        hist = None if L == 0 else history.to(self.device, torch.int32).t().contiguous()     # kernel layout: [L][B]
        tok = torch.empty(B, dtype=torch.int32, device=self.device)
        scores = torch.empty(B, V, dtype=torch.float32, device=self.device) if return_scores else None
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_op_sample(N.ptr(lg), B, V, N.ptr(hist), L, C.byref(spec), N.ptr(tok), N.ptr(scores), self._stream()), "vcla_op_sample")
        return tok, scores

    # ---- beam search (include/vcla.h, "beam search") --------------------------------------------------------
    _beam = None

    @staticmethod
    def beam_spec(num_beams, max_new_tokens, length_penalty=1.0, early_stopping=False, eos_token_id=(), repetition_penalty=1.0,
                  no_repeat_ngram_size=0, min_new_tokens=0) -> "N.VclaBeam":
        eos = list(eos_token_id)
        es = 2 if early_stopping == "never" else (1 if early_stopping is True else 0)
        arr = (C.c_int * 4)(*(eos + [0] * (4 - len(eos)))[:4])
        return N.VclaBeam(int(num_beams), float(length_penalty), es, int(max_new_tokens), len(eos), arr, float(repetition_penalty),
                          int(no_repeat_ngram_size or 0), int(min_new_tokens or 0))

    def set_beam(self, spec: Optional["N.VclaBeam"]):
        """spec = beam_spec(...): prefill forks every prompt to num_beams rows and decode steps run the beam kernels; None: off."""
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_set_beam(self._ctx, C.byref(spec) if spec is not None else None), "vcla_set_beam")
        self._beam = spec

    # ---- fan-out: n sampled replies per prompt from one prefill (include/vcla.h, "fan-out") -------------------------------------
    _fanout = 1

    def set_fanout(self, n: int):
        """n > 1: prefill forks every prompt to n rows sharing its KV pages (row b * n + j), the first pick drawn per row; 1: off."""
        N.check(self.lib.vcla_set_fanout(self._ctx, int(n)), "vcla_set_fanout")
        self._fanout = int(n)

    def read_beams(self, items: int):
        """-> (tokens (items, K, max_new) int32, lengths (items, K), scores (items, K) f32, done (items,)) host tensors: the finished-
        hypothesis store of the resident beam search, best first."""
        K, n = self._beam.num_beams, self._beam.max_new_tokens
        tok = torch.zeros(items, K, n, dtype=torch.int32)
        lens = torch.zeros(items, K, dtype=torch.int32)
        scores = torch.zeros(items, K, dtype=torch.float32)
        done = torch.zeros(items, dtype=torch.int32)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_beams(self._ctx, N.ptr(tok), N.ptr(lens), N.ptr(scores), N.ptr(done)), "vcla_read_beams")
        return tok, lens, scores, done

    def read_beam_done(self, items: int) -> torch.Tensor:
        done = torch.zeros(items, dtype=torch.int32)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_beams(self._ctx, None, None, None, N.ptr(done)), "vcla_read_beams")
        return done

    def beam_cow_bytes(self, reset: bool = False) -> int:
        v = C.c_int64()
        N.check(self.lib.vcla_beam_cow_bytes(self._ctx, C.byref(v), 1 if reset else 0), "vcla_beam_cow_bytes")
        return v.value

    def op_beam_step(self, logits: torch.Tensor, history: Optional[torch.Tensor], t: int, spec: "N.VclaBeam", state: dict) -> dict:
        """The two beam-selection kernels on caller data.  logits (rows, V) f32 (t == 0: the B prompts, else B * K beams); history
        (rows, t) tokens; state: dict of CUDA tensors run (B*K,) f32, scores (B,K) f32, lens / fin (B,K) int32, tokens (B,K,max_new)
        int32, items (B,2) int32 -- created by the call at t == 0, updated in place.  -> {parent, token (B*K,), cand (B,M,2)}."""
        lg = logits.to(self.device, torch.float32).contiguous()
        rows, V = lg.shape
        K, n = spec.num_beams, spec.max_new_tokens
        B = rows if t == 0 else rows // K
        M = max(2, 1 + spec.n_eos) * K
        dev = self.device
        if t == 0:
            state.update(run=torch.zeros(B * K, dtype=torch.float32, device=dev), scores=torch.zeros(B, K, dtype=torch.float32, device=dev),
                         lens=torch.zeros(B, K, dtype=torch.int32, device=dev), fin=torch.zeros(B, K, dtype=torch.int32, device=dev),
                         tokens=torch.zeros(B, K, n, dtype=torch.int32, device=dev), items=torch.zeros(B, 2, dtype=torch.int32, device=dev))
        hist = None if t == 0 else history.to(dev, torch.int32).t().contiguous()      # kernel layout: [t][rows]
        parent = torch.empty(B * K, dtype=torch.int32, device=dev)
        token = torch.empty(B * K, dtype=torch.int32, device=dev)
        cand = torch.empty(B, M, 2, dtype=torch.int32, device=dev)
        s = state
        with torch.cuda.device(dev):
            N.check(self.lib.vcla_op_beam_step(N.ptr(lg), B, V, N.ptr(hist), t, C.byref(spec), N.ptr(s["run"]), N.ptr(s["scores"]), N.ptr(s["lens"]),
                                               N.ptr(s["fin"]), N.ptr(s["tokens"]), N.ptr(s["items"]), N.ptr(parent), N.ptr(token), N.ptr(cand),
                                               self._stream()), "vcla_op_beam_step")
        return dict(parent=parent, token=token, cand=cand)

    # ---- token streaming (include/vcla.h, "token streaming") ---------------------------------------------------------------
    def stream_supported(self) -> bool:
        return True

    def stream_arm(self, on: bool):
        """Armed, every token choice (prefill / extend pick, each decode step) publishes its step into the host ring."""
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_stream_arm(self._ctx, 1 if on else 0), "vcla_stream_arm")

    def stream_wait(self, target: int, timeout_us: int = -1) -> int:
        """-> steps published so far, >= target unless the timeout (microseconds, < 0: none) expired first.  Raises when all armed
        work has completed and step `target` was never published.  The GIL is released while it waits."""
        n = C.c_int()
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_stream_wait(self._ctx, int(target), int(timeout_us), C.byref(n)), "vcla_stream_wait")
        return n.value

    def stream_read(self, lo: int, hi: int, B: int) -> torch.Tensor:
        """(hi - lo, B) int32 host tensor: the tokens of published steps lo..hi-1."""
        out = torch.empty(hi - lo, B, dtype=torch.int32)
        if hi > lo:
            N.check(self.lib.vcla_stream_read(self._ctx, int(lo), int(hi), int(B), N.ptr(out)), "vcla_stream_read")
        return out

    def read_history(self, B: int, n_steps: int) -> torch.Tensor:
        """(n_steps, B) int32 CUDA tensor: tokens chosen by the prefill (row 0) and each decode step since."""
        out = torch.empty(n_steps, B, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_history(self._ctx, N.ptr(out), B, n_steps, self._stream()), "vcla_read_history")
        return out

    def reset(self):
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_reset(self._ctx, self._stream()), "vcla_reset")

    # ---- paged KV cache introspection ---------------------------------------------------------
    def kv_geometry(self) -> Tuple[int, int, int]:
        """(pages per sequence, pages in the pool, tokens per page)."""
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        N.check(self.lib.vcla_kv_geometry(self._ctx, C.byref(a), C.byref(b), C.byref(c)), "vcla_kv_geometry")
        return a.value, b.value, c.value

    def kv_read_layer(self, layer: int) -> torch.Tensor:
        """One layer's pool bytes (uint8, host): bf16 rows [pages][K|V][heads][page_tokens][128], or with the int8 cache the int8 rows in
        that order followed by their fp32 scales (include/vcla.h).  Synchronises the device."""
        out = torch.empty(self.memory_bytes()[1] // self.path_cfg["t_layers"], dtype=torch.uint8)
        N.check(self.lib.vcla_kv_read_layer(self._ctx, int(layer), N.ptr(out)), "vcla_kv_read_layer")
        return out

    def kv_pages(self):
        """-> (page_table (max_batch, pages_per_seq) int32, pages owned per sequence (max_batch,), free pages, exhausted flag)."""
        pps, _total, _pt = self.kv_geometry()
        table = torch.zeros(self.max_batch, pps, dtype=torch.int32)
        owned = torch.zeros(self.max_batch, dtype=torch.int32)
        state = torch.zeros(2, dtype=torch.int32)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_kv_read_pages(self._ctx, N.ptr(table), N.ptr(owned), N.ptr(state)), "vcla_kv_read_pages")
        return table, owned, int(state[0]), int(state[1])

    def kv_debug_shuffle(self, seed: int):
        self.session += 1
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_kv_debug_shuffle(self._ctx, seed), "vcla_kv_debug_shuffle")

    def kernel_launches(self, reset: bool = False) -> int:
        return int(self.lib.vcla_kernel_launches(self._ctx, 1 if reset else 0))

    def bench_decode_gemm(self, which: int, B: int, reps: int = 3):
        """(mean microseconds per launch, weight bytes per launch) of one decode GEMM shape; see vcla.h."""
        us, nbytes = C.c_float(), C.c_int64()
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_bench_decode_gemm(self._ctx, which, B, reps, C.byref(us), C.byref(nbytes), self._stream()), "vcla_bench_decode_gemm")
        return us.value, nbytes.value

    def trace_enable(self, max_events: int = 4096):
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_trace_enable(self._ctx, max_events), "vcla_trace_enable")

    def trace_read(self, max_events: int = 4096):
        """-> list of (tag, t_entry_ns, t_dep_ns, t_exit_ns) recorded since the last read."""
        buf = torch.zeros(max_events, 4, dtype=torch.int64)
        n = C.c_int()
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_trace_read(self._ctx, N.ptr(buf), max_events, C.byref(n)), "vcla_trace_read")
        return [tuple(int(x) for x in row) for row in buf[: n.value].tolist()]

    def read_stage(self, stage: str, B: int) -> torch.Tensor:
        c = self.path_cfg
        shapes = {"vit_out": (B, (c["v_image"] // c["v_patch"]) ** 2 + 1, c["v_hidden"]),
                  "post_ln": (B, (c["v_image"] // c["v_patch"]) ** 2 + 1, c["v_hidden"]),
                  "resampler_out": (B, c["r_queries"], c["r_hidden"]),
                  "projector_out": (B, c["r_queries"], c["t_hidden"]),
                  "step_logits": (B, c["t_vocab"]), "lookup_tokens": (B,)}
        out = torch.empty(shapes[stage], dtype=torch.float32)
        with torch.cuda.device(self.device):
            N.check(self.lib.vcla_read_stage(self._ctx, stage.encode(), B, N.ptr(out), self._stream()), f"vcla_read_stage({stage})")
        return out
