"""Host-side driver of the H100 lookahead/verification step.

One ``LookaheadEngine`` wraps one HF ``LlamaForCausalLM`` (or ``Qwen3ForCausalLM``, whose per-head q/k RMSNorm
runs inside ``lade_rope_append_qknorm``, or ``Qwen2ForCausalLM``, whose q/k/v projection biases are added to the fp32
QKV projection inside ``lade_rope_append_bias``) on one GPU.  Per decoding step it launches
(through the C-ABI of ``include/lade_sm100.h``):

    lade_step_layout -> embedding gather -> L x [ lade_rmsnorm -> QKV GEMM -> lade_rope_append ->
    lade_attn_fwd -> O GEMM -> lade_rmsnorm(+residual) -> gate/up GEMM -> lade_swiglu -> down GEMM ]
    -> lade_rmsnorm_gather (live lm_head rows only) -> lm_head GEMM -> lade_argmax_rows ->
    lade_accept_update -> lade_kv_compact [-> lade_capture_rows, with capture_logits]

which is the GPU re-design of one iteration of the reference's ``while True`` loop
(``lade/decoding.py:923-1219``) including ``jforward_multilevel``
(``lade/models/modeling_llama.py:1381-1608``).  The dense projections are plain library GEMMs
(cuBLAS through ``torch.mm``); everything else is this repo's CUDA.  All per-step scalars live in
device memory, so the steady step is a fixed-shape launch sequence that is captured once in a CUDA
graph and replayed; the host reads back one 48-int record per step (accepted tokens + done flag).

PyTorch is used for device memory, streams and the GEMMs only.  There is no CPU fallback: a missing
library or a non-CUDA model raises.
"""
from __future__ import annotations

import ctypes as C
import random
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _cabi
from ._cabi import LadeConfig, LadeError, check


@dataclass
class StepRecord:
    n_emit: int
    max_hit: int
    hits: List[int]
    n_guess: int
    kv_len: int
    done: bool


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


_PROC_KEYS = ("penalty", "prompt_ignore_length", "ngram_size", "min_length", "eos_token_id")


def processors_record(processors: dict) -> _cabi.LadeProcessors:
    """The LadeProcessors record of a `processors` dict (see LookaheadEngine.generate).  The penalty is rounded to fp32
    as torch does for a python scalar on a float32 tensor."""
    unknown = set(processors) - set(_PROC_KEYS)
    if unknown:
        raise LadeError(f"unknown logits-processor fields {sorted(unknown)} (known: {', '.join(_PROC_KEYS)})")
    r = _cabi.LadeProcessors()
    if processors.get("penalty") is not None:
        p = np.float32(processors["penalty"])
        if not (np.isfinite(p) and p > 0):
            raise LadeError(f"repetition penalty must be finite and > 0 (got {processors['penalty']})")
        r.flags |= _cabi.PROC_REPETITION_PENALTY
        r.penalty_bits = int(p.view(np.uint32))
        r.prompt_ignore_length = int(processors.get("prompt_ignore_length") or 0)
        if r.prompt_ignore_length < 0:
            raise LadeError("prompt_ignore_length must be >= 0")
    if processors.get("ngram_size") is not None:
        n = int(processors["ngram_size"])
        if not 1 <= n <= _cabi.PROC_MAX_NGRAM:
            raise LadeError(f"no_repeat_ngram_size must be in 1..{_cabi.PROC_MAX_NGRAM} on device (got {n})")
        r.flags |= _cabi.PROC_NO_REPEAT_NGRAM
        r.ngram_size = n
    eos = [int(e) for e in (processors.get("eos_token_id") or ())]
    if processors.get("min_length") is not None and eos:
        if len(eos) > _cabi.PROC_MAX_EOS:
            raise LadeError(f"at most {_cabi.PROC_MAX_EOS} eos ids for the min-length processors (got {len(eos)})")
        r.flags |= _cabi.PROC_MIN_LENGTH
        r.eos_bound = int(processors["min_length"])
        r.n_eos = len(eos)
        for i, e in enumerate(eos):
            r.eos_token_id[i] = e
    return r


def first_matching_candidate(guess_tokens: Sequence[int], gs: int, hits: Sequence[int], i: int) -> int:
    """The candidate the sampling verification accepted at position i: the lowest-index n-gram whose tokens 0..i equal
    hits[0..i] (an earlier n-gram carrying hits[i] would have been tested first, and its rejection zeroes that token
    for every later one), or -1 when none does (hits[i] was drawn, not accepted)."""
    for e in range(len(guess_tokens) // gs):
        if all(guess_tokens[e * gs + u] == hits[u] for u in range(i + 1)):
            return e
    return -1


def decided_slots(n_emit: int, hits: Sequence[int], window_cap: int, gs: int, sampling: bool, max_hit_idx: int = 0,
                  guess_tokens: Sequence[int] = ()) -> List[int]:
    """The lm slot each of a step's n_emit emitted tokens was decided from (what lade_capture_rows copies): slot 0 for
    the first; for token j >= 1 the verification slot (e, j-1), with e = max_hit_idx on the greedy path and the first
    matching candidate at position j-1 on the sampling path."""
    slots = [0] if n_emit > 0 else []
    for j in range(1, n_emit):
        e = first_matching_candidate(guess_tokens, gs, hits, j - 1) if sampling else max_hit_idx
        slots.append(1 + window_cap + e * gs + j - 1)
    return slots


def attn_kv_bound(max_total_len: int, q_nonprefill: int, level: int) -> int:
    """Upper bound of kv_len + q_len of any step an engine built for `max_total_len` runs, the surplus step
    generate() queues before it knows the generation has ended included.  A real step starts with at most
    max_length - 1 tokens out and emits up to N - 1 (a full accept), so the state it leaves holds at most
    max_length + N - 2 tokens and a cache of kv_len = n_out - 1 <= max_length + N - 3 rows; any step laid out on that
    state adds at most q_nonprefill rows.  generate() itself queues the surplus step only behind a step that starts
    at max_length - 2 tokens out or fewer, so the steps it launches stay one row below this bound (kv_len <=
    max_length + N - 4); the extra row keeps the bound valid for any step run on a finished state."""
    return max_total_len + level - 3 + q_nonprefill


class LookaheadEngine:
    """Device-resident lookahead decoding for one Llama-shaped model (batch 1, bf16 or fp16, CUDA): Llama, Qwen3 with
    its per-head q/k RMSNorm, or Qwen2 / Qwen2.5 with biases on q_proj, k_proj and v_proj (o_proj and the MLP without).
    On a model with those biases the QKV projection is written in fp32 and the bias is added to that accumulator before
    the single rounding to the model dtype, as nn.Linear's addmm does."""

    def __init__(self, model, window_size: int, level: int, guess_set_size: int,
                 pool_from_prompt: bool = False, max_total_len: int = 4096, attn_impl: int = 0,
                 attn_splits: Optional[int] = None, use_cuda_graph: bool = True,
                 dist_workers: int = 1, rank: int = 0, process_group=None, pipeline_host: bool = True):
        self.lib = _cabi.load()
        self.pipeline_host = bool(pipeline_host)
        cfg = model.config
        p0 = next(model.parameters())
        if p0.device.type != "cuda":
            raise LadeError("LookaheadEngine needs the model on a CUDA device (no CPU fallback)")
        if p0.dtype not in (torch.bfloat16, torch.float16):
            raise LadeError(f"LookaheadEngine supports bf16 and fp16 models (got {p0.dtype})")
        # element type of the model: every kernel exists per dtype (bf16: the unsuffixed C-ABI entry points, fp16: *_f16)
        self.dt = p0.dtype
        sfx = "" if self.dt == torch.bfloat16 else "_f16"
        self.k_rmsnorm = getattr(self.lib, "lade_rmsnorm" + sfx)
        self.k_rmsnorm_gather = getattr(self.lib, "lade_rmsnorm_gather" + sfx)
        self.k_rope_append = getattr(self.lib, "lade_rope_append" + sfx)
        self.k_rope_append_qknorm = getattr(self.lib, "lade_rope_append_qknorm" + sfx)
        self.k_rope_append_bias = getattr(self.lib, "lade_rope_append_bias" + sfx)
        self.k_swiglu = getattr(self.lib, "lade_swiglu" + sfx)
        self.k_argmax_rows = getattr(self.lib, "lade_argmax_rows" + sfx)
        self.k_argmax_processed = getattr(self.lib, "lade_argmax_processed" + sfx)
        self.k_attn_fwd = getattr(self.lib, "lade_attn_fwd" + sfx)
        self.k_sample_verify = getattr(self.lib, "lade_sample_verify" + sfx)
        self.k_sample_verify_warped = getattr(self.lib, "lade_sample_verify_warped" + sfx)
        self.k_capture_rows = getattr(self.lib, "lade_capture_rows" + sfx)
        if level < 3:
            raise LadeError("LEVEL must be >= 3 (lade/decoding.py:902)")
        if guess_set_size == -1:
            raise LadeError("GUESS_SET_SIZE=-1 (unbounded python set) is not supported on device")
        self.model = model
        self.dev = p0.device
        self.W, self.N, self.G = int(window_size), int(level), int(guess_set_size)
        self.GS = self.N - 1
        self.WCAP = self.W + self.N - 3
        self.pool_from_prompt = bool(pool_from_prompt)
        self.H = cfg.hidden_size
        self.L = cfg.num_hidden_layers
        self.nh = cfg.num_attention_heads
        self.nkv = getattr(cfg, "num_key_value_heads", None) or self.nh
        self.D = getattr(cfg, "head_dim", None) or self.H // self.nh
        self.I = cfg.intermediate_size
        self.V = cfg.vocab_size
        self.eps = float(cfg.rms_norm_eps)
        if self.D not in (64, 128):
            raise LadeError(f"head_dim {self.D} unsupported (attention kernels are instantiated for 128 and 64)")
        self.max_pos = int(getattr(cfg, "max_position_embeddings", 4096))
        rp = getattr(cfg, "rope_parameters", None) or {}
        rope_type = (rp.get("rope_type") if isinstance(rp, dict) else None) or "default"
        legacy = getattr(cfg, "rope_scaling", None)
        if isinstance(legacy, dict) and (legacy.get("rope_type") or legacy.get("type") or "default") != "default":
            rope_type = legacy.get("rope_type") or legacy.get("type")
        if rope_type != "default":
            # the reference knows "linear" / "dynamic" NTK scaling (modeling_llama.py:271-318); neither is wired into the
            # device RoPE tables here, and silently decoding with unscaled positions would be wrong
            raise LadeError(f"rope scaling '{rope_type}' is not supported (only the default rotary embedding)")
        self.rope_theta = float(rp.get("rope_theta", getattr(cfg, "rope_theta", 10000.0)) if isinstance(rp, dict)
                                else getattr(cfg, "rope_theta", 10000.0))
        self._check_attention_layout(model, int(max_total_len))
        self.has_qkv_bias = self._check_biases(model)
        self.attn_impl = attn_impl
        self.use_cuda_graph = use_cuda_graph
        self.lm_cap = 1 + self.WCAP + self.G * self.GS
        # lookahead parallelism (lade_distributed): full replica per rank, window/guess slices per rank
        self.DW = int(dist_workers) if dist_workers and dist_workers > 1 else 1
        self.rank = int(rank) if self.DW > 1 else 0
        self.pg = process_group
        if self.DW > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                raise LadeError("DIST_WORKERS > 1 needs an initialised torch.distributed process group")
            if dist.get_world_size(self.pg) != self.DW:
                raise LadeError("DIST_WORKERS config should be equal to work size")      # lade/utils.py:33
        self._nccl_comm = C.c_void_p()
        if self.DW > 1:
            self._lp_comm_create()
        self.max_total_len = int(max_total_len)
        probe = self._make_config(())
        self.q_steady = int(self.lib.lade_step_rows_bound(C.byref(probe), 1, self.N))    # fixed steady shape
        self.rec_ints = int(self.lib.lade_lp_record_ints(C.byref(probe)))
        sm = torch.cuda.get_device_properties(self.dev).multi_processor_count
        q_tiles = (self.q_steady + 127) // 128
        # one CTA per SM (shared-memory bound): keep the split grid within a single wave
        self.attn_splits = int(attn_splits) if attn_splits else max(1, min(8, sm // (self.nh * q_tiles)))   # <= 8: the splits of a head form a thread-block cluster

        # non-prefill steps: the steady shape, or a window-fill step when it is larger (G = 0 and W < N-2 ...)
        self.q_nonprefill = max([self.q_steady] + [int(self.lib.lade_step_rows_bound(C.byref(probe), 1, k))
                                                   for k in range(1, self.N - 1)])
        self.kv_capacity = self.max_total_len + self.q_nonprefill + self.WCAP + 8
        # kv_bound of lade_attn_fwd: an upper bound of kv_len + q_len over the whole generation.  Only impl 3 (the
        # reference-order variant, every K/V tile of a split resident in shared memory) needs a tight one: at most
        # 3 KV tiles of 128 rows per split and 8 splits per head
        self.attn_kv_bound = self.kv_capacity
        if self.attn_impl == 3:
            self.attn_kv_bound = min(self.kv_capacity, attn_kv_bound(self.max_total_len, self.q_nonprefill, self.N))
            need = -(-((self.attn_kv_bound + 127) // 128) // 3)
            if need > 8:
                raise LadeError(f"attn_impl=3 holds at most 3072 rows of context (asked for {self.attn_kv_bound}: "
                                f"max_total_len {self.max_total_len} + N - 3 = {self.N - 3} rows a final accept may "
                                f"overshoot + {self.q_nonprefill} step rows)")
            if not attn_splits:
                self.attn_splits = max(self.attn_splits, need)
            elif self.attn_splits < need:
                raise LadeError(f"attn_impl=3 needs attn_splits >= {need} for {self.attn_kv_bound} rows of context")
        self._fuse_weights()
        self._rope_tables()
        self._alloc(self.q_nonprefill)
        self._ctx = C.c_void_p()
        self._lcfg = None
        self._graph = None
        self._pinned_res = torch.empty(_cabi.RES_INTS, dtype=torch.int32, pin_memory=True)
        # two result slots + events: the host reads step i's record while step i+1 is already queued on the GPU
        self._pinned_ring = [torch.empty(_cabi.RES_INTS, dtype=torch.int32, pin_memory=True) for _ in range(2)]
        self._res_events = [torch.cuda.Event() for _ in range(2)]
        # greedy logits processors of the current generate() (LadeProcessors, written by begin()); off: plain argmax
        self.proc_dev = torch.zeros(C.sizeof(_cabi.LadeProcessors) // 4, dtype=torch.int32, device=self.dev)
        self.processors_on = False
        self.launches = 0   # kernels of THIS repo launched (graph replays counted by their content)
        # tests set a device float[>= 2 + G*(N-1) + W]: lade_sample_verify then records the uniforms it consumed
        self.debug_uniforms: Optional[torch.Tensor] = None
        # tests set a device float[>= 1 + 2*(N-1)]: lade_sample_verify_warped then records each visited row's cut
        self.debug_cuts: Optional[torch.Tensor] = None
        # logits capture of the current generate() (capture_logits=True): [rows][V] in the model dtype, row r = the lm
        # row generated token r was decided from (lade_capture_rows after every step's commit)
        self.capture_on = False
        self.capture_buf: Optional[torch.Tensor] = None
        self.last_logits: Optional[torch.Tensor] = None
        self.last_steps = 0
        self.last_records: List[StepRecord] = []

    # ------------------------------------------------------------------------------------------
    def _check_attention_layout(self, model, max_total_len: int) -> None:
        """Per-head q/k RMSNorm (Qwen3Attention: q_norm / k_norm in front of the rotary embedding) and sliding-window
        layers.  A model with both norms on every layer, each of weight [head_dim], runs with the norms fused into the
        RoPE kernel; any other shape of them, or a layer HF would run with a sliding window shorter than the engine's
        capacity, is refused here, before anything is allocated: decoding it with the Llama step would be wrong."""
        cfg = model.config
        layer_types = getattr(cfg, "layer_types", None) or ()
        window = getattr(cfg, "sliding_window", None)
        if "sliding_attention" in layer_types and window is not None and int(window) < max_total_len:
            raise LadeError(f"sliding-window attention (sliding_window={window} < max_total_len={max_total_len} on "
                            f"{list(layer_types).count('sliding_attention')} layers) is not supported")
        self.q_norm_w: Optional[List[torch.Tensor]] = None
        self.k_norm_w: Optional[List[torch.Tensor]] = None
        self.qk_eps: List[float] = []
        found = [(getattr(l.self_attn, "q_norm", None), getattr(l.self_attn, "k_norm", None)) for l in model.model.layers]
        if all(q is None and k is None for q, k in found):
            return
        qw, kw = [], []
        for li, (qn, kn) in enumerate(found):
            if qn is None or kn is None:
                raise LadeError(f"layer {li} has {'k_norm' if qn is None else 'q_norm'} without "
                                f"{'q_norm' if qn is None else 'k_norm'}: not supported")
            for name, m_ in (("q_norm", qn), ("k_norm", kn)):
                w = getattr(m_, "weight", None)
                if w is None or tuple(w.shape) != (self.D,) or w.dtype != self.dt or not w.is_contiguous() \
                        or not hasattr(m_, "variance_epsilon"):
                    raise LadeError(f"layer {li} {name} ({type(m_).__name__}, weight "
                                    f"{None if w is None else (tuple(w.shape), w.dtype)}) is not an RMSNorm over each "
                                    f"head of {self.D} in {self.dt}: only per-head q/k norms (Qwen3) are supported")
            if float(qn.variance_epsilon) != float(kn.variance_epsilon):
                raise LadeError(f"layer {li}: q_norm and k_norm have different eps: not supported")
            qw.append(qn.weight)
            kw.append(kn.weight)
            self.qk_eps.append(float(qn.variance_epsilon))
        self.q_norm_w, self.k_norm_w = qw, kw

    def _check_biases(self, model) -> bool:
        """True for a model whose q_proj, k_proj and v_proj carry a bias on every layer (Qwen2 / 2.5), False for one
        without any projection bias.  Every other placement of biases is refused here, before anything is allocated:
        the step adds biases to q, k and v only."""
        q_norms = self.q_norm_w is not None
        n_biased = 0
        for li, layer in enumerate(model.model.layers):
            a, mlp = layer.self_attn, layer.mlp
            if getattr(a.o_proj, "bias", None) is not None:
                raise LadeError(f"layer {li}: o_proj has a bias (Llama attention_bias=True): not supported")
            if any(getattr(m_, "bias", None) is not None for m_ in (mlp.gate_proj, mlp.up_proj, mlp.down_proj)):
                raise LadeError(f"layer {li}: MLP bias (mlp_bias=True) is not supported")
            have = [getattr(getattr(a, n_), "bias", None) is not None for n_ in ("q_proj", "k_proj", "v_proj")]
            if not any(have):
                continue
            if not all(have):
                missing = [n_ for n_, h_ in zip(("q_proj", "k_proj", "v_proj"), have) if not h_]
                raise LadeError(f"layer {li}: a bias on only some of q/k/v ({', '.join(missing)} without): not supported")
            for n_ in ("q_proj", "k_proj", "v_proj"):
                m_ = getattr(a, n_)
                b = m_.bias
                if b.dtype != self.dt or tuple(b.shape) != (m_.weight.shape[0],) or b.device != m_.weight.device:
                    raise LadeError(f"layer {li}: {n_} bias {(tuple(b.shape), b.dtype)} is not "
                                    f"[{m_.weight.shape[0]}] in {self.dt}: not supported")
            if q_norms:
                raise LadeError(f"layer {li}: q/k/v biases together with per-head q/k norms are not supported")
            n_biased += 1
        if 0 < n_biased < len(model.model.layers):
            raise LadeError(f"q/k/v biases on {n_biased} of {len(model.model.layers)} layers: not supported")
        return n_biased > 0

    def _fuse_weights(self):
        """Fuse q/k/v and gate/up into single GEMM operands (and the q/k/v biases into one vector); re-point the HF
        parameters at views of the fused storage so no second copy of the weights stays resident."""
        m = self.model.model
        self.embed = m.embed_tokens.weight
        self.norm_w = m.norm.weight
        self.lm_head = self.model.lm_head.weight
        self.w_qkv, self.w_o, self.w_gu, self.w_down, self.ln1, self.ln2 = [], [], [], [], [], []
        self.b_qkv: Optional[List[torch.Tensor]] = [] if self.has_qkv_bias else None
        # a previous engine of this model already fused: reuse its storage (no second 13 GB transient) as long as
        # the HF parameters still point into it
        prev = self.model.__dict__.get("_lade_fused")
        with torch.no_grad():
            for li, layer in enumerate(m.layers):
                a, mlp = layer.self_attn, layer.mlp
                nq, nk = a.q_proj.weight.shape[0], a.k_proj.weight.shape[0]
                qkv = gu = bqkv = None
                if prev is not None and li < len(prev[0]):
                    pq, pg = prev[0][li], prev[1][li]
                    pb = prev[2][li] if self.has_qkv_bias and len(prev) > 2 and li < len(prev[2]) else None
                    if (pq.data_ptr() == a.q_proj.weight.data_ptr() and pq[nq:].data_ptr() == a.k_proj.weight.data_ptr()
                            and pq[nq + nk:].data_ptr() == a.v_proj.weight.data_ptr()
                            and pg.data_ptr() == mlp.gate_proj.weight.data_ptr()
                            and pg[self.I:].data_ptr() == mlp.up_proj.weight.data_ptr()
                            and (not self.has_qkv_bias or (
                                pb is not None and pb.data_ptr() == a.q_proj.bias.data_ptr()
                                and pb[nq:].data_ptr() == a.k_proj.bias.data_ptr()
                                and pb[nq + nk:].data_ptr() == a.v_proj.bias.data_ptr()))):
                        qkv, gu, bqkv = pq, pg, pb
                if qkv is None:
                    qkv = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], dim=0).contiguous()
                    a.q_proj.weight.data = qkv[:nq]
                    a.k_proj.weight.data = qkv[nq:nq + nk]
                    a.v_proj.weight.data = qkv[nq + nk:]
                    gu = torch.cat([mlp.gate_proj.weight, mlp.up_proj.weight], dim=0).contiguous()
                    mlp.gate_proj.weight.data = gu[: self.I]
                    mlp.up_proj.weight.data = gu[self.I:]
                    if self.has_qkv_bias:
                        bqkv = torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]).contiguous()
                        a.q_proj.bias.data = bqkv[:nq]
                        a.k_proj.bias.data = bqkv[nq:nq + nk]
                        a.v_proj.bias.data = bqkv[nq + nk:]
                self.w_qkv.append(qkv)
                if self.has_qkv_bias:
                    self.b_qkv.append(bqkv)
                self.w_gu.append(gu)
                self.w_o.append(a.o_proj.weight)
                self.w_down.append(mlp.down_proj.weight)
                self.ln1.append(layer.input_layernorm.weight)
                self.ln2.append(layer.post_attention_layernorm.weight)
        self.model.__dict__["_lade_fused"] = (self.w_qkv, self.w_gu, self.b_qkv or [])

    def _rope_tables(self):
        # fp32 math then cast to the model dtype: lade/models/modeling_llama.py:240-256,:264-265
        D = self.D
        inv_freq = 1.0 / (self.rope_theta ** (torch.arange(0, D, 2).float() / D))
        # the reference regrows its table on demand (:258-261); size ours for the longest sequence
        self.table_len = max(self.max_pos, self.max_total_len + self.WCAP + self.N + 8)
        t = torch.arange(self.table_len, dtype=inv_freq.dtype)
        freqs = torch.outer(t, inv_freq)
        emb = torch.cat((freqs, freqs), dim=-1)
        self.cos = emb.cos().to(self.dt).to(self.dev).contiguous()
        self.sin = emb.sin().to(self.dt).to(self.dev).contiguous()

    def _alloc(self, rows: int):
        dev, bf = self.dev, self.dt
        self.rows_cap = rows
        i32 = dict(dtype=torch.int32, device=dev)
        self.ids = torch.zeros(rows, **i32)
        self.pos = torch.zeros(rows, **i32)
        self.rowdesc = torch.zeros(rows, **i32)
        self.mask_words = (max(self.q_nonprefill, 32) + 31) // 32 + 1      # non-prefill steps are short
        self.rowmask = torch.zeros(self.mask_words * 32 * self.mask_words, **i32)
        self.meta = torch.zeros(_cabi.META_INTS, **i32)
        self.lm_rows = torch.zeros(self.lm_cap, **i32)
        self.am = torch.zeros(self.lm_cap, **i32)
        self.res = torch.zeros(_cabi.RES_INTS, **i32)
        self.dec_dev = torch.zeros(self.rec_ints + 4 + self.W, **i32)          # decision record of the sampling path
        if not hasattr(self, "rng_state"):
            self.rng_state = torch.zeros(2, dtype=torch.int64, device=dev)     # Philox (seed, offset), advanced on device
            self.sample_temperature, self.sample_top_k, self.sample_top_p = 1.0, 0, 1.0
            self.sample_min_p, self.sample_epsilon, self.sample_eta = 0.0, 0.0, 0.0
        self.lp_send = torch.zeros(self.rec_ints, **i32)
        self.lp_recv = torch.zeros(self.DW * self.rec_ints, **i32)
        self.h = torch.empty(rows, self.H, dtype=bf, device=dev)
        self.xn = torch.empty(rows, self.H, dtype=bf, device=dev)
        # a model with q/k/v biases: the QKV projection's fp32 accumulator, which lade_rope_append_bias adds the bias to
        # and rounds once
        self.qkv = torch.empty(rows, (self.nh + 2 * self.nkv) * self.D, dtype=torch.float32 if self.has_qkv_bias else bf,
                               device=dev)
        self.qb = torch.zeros(self.nh, rows, self.D, dtype=bf, device=dev)
        self.attn_out = torch.empty(rows, self.nh * self.D, dtype=bf, device=dev)
        self.o_buf = torch.empty(rows, self.H, dtype=bf, device=dev)
        self.gu = torch.empty(rows, 2 * self.I, dtype=bf, device=dev)
        self.act = torch.empty(rows, self.I, dtype=bf, device=dev)
        self.d_buf = torch.empty(rows, self.H, dtype=bf, device=dev)
        self.xn_lm = torch.empty(self.lm_cap, self.H, dtype=bf, device=dev)
        self.logits = torch.empty(self.lm_cap, self.V, dtype=bf, device=dev)
        if not hasattr(self, "kv"):
            self.kv = torch.zeros(self.L, 2, self.nkv, self.kv_capacity, self.D, dtype=bf, device=dev)
        nbytes = self.lib.lade_attn_scratch_bytes(rows, self.nh, self.D, self.attn_splits)
        self.attn_scratch = torch.zeros(int(nbytes), dtype=torch.uint8, device=dev)

    # ------------------------------------------------------------------------------------------
    def _make_config(self, eos_ids) -> LadeConfig:
        c = LadeConfig()
        c.window_size, c.level, c.guess_set_size = self.W, self.N, self.G
        c.pool_from_prompt = int(self.pool_from_prompt)
        c.vocab_size = self.V
        c.max_total_len = self.max_total_len + self.N + 8
        c.n_eos = len(eos_ids)
        for i, e in enumerate(eos_ids):
            c.eos_token_id[i] = int(e)
        c.dist_workers, c.rank = self.DW, self.rank
        return c

    def _ensure_ctx(self, eos_ids: Sequence[int]):
        eos_ids = list(eos_ids)
        if len(eos_ids) > 4:
            raise LadeError(f"at most 4 eos_token_id values are supported on device (got {len(eos_ids)})")
        key = (tuple(eos_ids),)
        if self._lcfg is not None and self._ctx_key == key:
            return
        if self._ctx:
            self.lib.lade_ctx_destroy(self._ctx)
            self._ctx = C.c_void_p()
            self._graph = None
        c = self._make_config(eos_ids)
        check(self.lib.lade_ctx_create(C.byref(c), C.byref(self._ctx)), "lade_ctx_create")
        self._lcfg = c
        self._ctx_key = key

    def close(self):
        if getattr(self, "_ctx", None):
            self.lib.lade_ctx_destroy(self._ctx)
            self._ctx = C.c_void_p()
        if getattr(self, "_nccl_comm", None):
            torch.cuda.synchronize(self.dev)
            self._graph = None
            self.lib.lade_nccl_comm_destroy(self._nccl_comm)
            self._nccl_comm = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------
    def _launch_step(self, rows: int, stream: int, commit: bool = True, prefill: bool = False):
        """All launches of one step on `stream` (the current stream) for `rows` materialised rows (rows <= rows_cap).
        Returns how many of this library's kernels were launched.  Each kernel family is a stage method below, so a
        tool can replace one stage on its own engine instance."""
        # prefill (step 0) is plain causal and carries no rowmask; every later step has one and must fit it
        mw = 0 if prefill else self.mask_words
        if mw and rows > (mw - 1) * 32:
            raise LadeError(f"step of {rows} rows does not fit the {mw}-word row mask")
        check(self.lib.lade_step_layout(self._ctx, stream, rows, _ptr(self.ids), _ptr(self.pos), _ptr(self.rowdesc),
                                        _ptr(self.lm_rows), _ptr(self.meta), _ptr(self.rowmask) if mw else 0, mw),
              "lade_step_layout"); n = 1
        h = self.h[:rows]
        torch.index_select(self.embed, 0, self.ids[:rows], out=h)
        xn, qkv, attn_out = self.xn[:rows], self.qkv[:rows], self.attn_out[:rows]
        o_buf, gu, act, d_buf = self.o_buf[:rows], self.gu[:rows], self.act[:rows], self.d_buf[:rows]
        qb = self.qb if rows == self.rows_cap else self.qb.view(-1)[: self.nh * rows * self.D].view(self.nh, rows, self.D)
        delta = None
        for l in range(self.L):
            kc, vc = self.kv[l, 0], self.kv[l, 1]
            n += self._norm(stream, h, delta, self.ln1[l], xn, rows)
            n += self._proj(xn, self.w_qkv[l], qkv)
            n += self._rope_append(stream, l, qkv, qb, kc, vc, rows)
            n += self._attention(stream, l, qb, kc, vc, attn_out, rows, prefill)
            n += self._proj(attn_out, self.w_o[l], o_buf)
            n += self._norm(stream, h, o_buf, self.ln2[l], xn, rows)
            n += self._proj(xn, self.w_gu[l], gu)
            n += self._swiglu(stream, gu, act, rows)
            n += self._proj(act, self.w_down[l], d_buf)
            delta = d_buf
        check(self.k_rmsnorm_gather(stream, _ptr(h), _ptr(delta), _ptr(self.norm_w), _ptr(self.lm_rows),
                                      _ptr(self.xn_lm), self.lm_cap, self.H, self.eps), "lade_rmsnorm_gather"); n += 1
        n += self._proj(self.xn_lm, self.lm_head, self.logits)
        if self.processors_on:
            check(self.k_argmax_processed(self._ctx, stream, _ptr(self.logits), self.lm_cap, self.V, self.V,
                                          _ptr(self.proc_dev), _ptr(self.am)), "lade_argmax_processed")
        else:
            check(self.k_argmax_rows(stream, _ptr(self.logits), self.lm_cap, self.V, self.V, _ptr(self.am)),
                  "lade_argmax_rows")
        n += 1
        n += self._commit(stream, commit)
        return n + self._capture(stream, commit)

    def _norm(self, stream: int, h, delta, w, out, rows: int) -> int:
        """out = rmsnorm(h + delta) * w; with a delta the residual sum is also written back to h."""
        check(self.k_rmsnorm(stream, _ptr(h), _ptr(delta), _ptr(w), _ptr(h) if delta is not None else 0, _ptr(out),
                             rows, self.H, self.eps), "lade_rmsnorm")
        return 1

    def _proj(self, x, w, out) -> int:
        """out = x @ w^T for an nn.Linear weight `w` (every projection of the step, lm_head included).  An fp32 `out` (the
        QKV projection of a model with q/k/v biases) receives the fp32 accumulator, not rounded to the model dtype."""
        if out.dtype == x.dtype:
            torch.mm(x, w.t(), out=out)
        else:
            torch.mm(x, w.t(), out_dtype=out.dtype, out=out)
        return 0

    def _rope_append(self, stream: int, l: int, qkv, qb, kc, vc, rows: int) -> int:
        """RoPE on q and k of layer `l` (after their per-head RMSNorm, or the q/k/v bias, on a model that has one); q to
        the head-major `qb`, k and v appended to the layer's cache."""
        args = (stream, _ptr(qkv), _ptr(self.cos), _ptr(self.sin), _ptr(self.pos), _ptr(self.meta), _ptr(qb), _ptr(kc),
                _ptr(vc), rows, rows, self.nh, self.nkv, self.D, self.kv_capacity, self.table_len)
        if self.b_qkv is not None:
            check(self.k_rope_append_bias(*args, _ptr(self.b_qkv[l])), "lade_rope_append_bias")
        elif self.q_norm_w is None:
            check(self.k_rope_append(*args), "lade_rope_append")
        else:
            check(self.k_rope_append_qknorm(*args, _ptr(self.q_norm_w[l]), _ptr(self.k_norm_w[l]), self.qk_eps[l]),
                  "lade_rope_append_qknorm")
        return 1

    def _attention(self, stream: int, l: int, qb, kc, vc, out, rows: int, prefill: bool) -> int:
        """Lookahead attention of layer `l` over the cache and the step's rows (causal on prefill, row mask after)."""
        mw = 0 if prefill else self.mask_words
        check(self.k_attn_fwd(stream, _ptr(qb), _ptr(kc), _ptr(vc), _ptr(out), _ptr(self.rowmask) if mw else 0, mw,
                              _ptr(self.meta), _ptr(self.attn_scratch), rows, self.nh, self.nkv, self.D,
                              self.kv_capacity, self.attn_kv_bound, self.attn_splits, self.attn_impl), "lade_attn_fwd")
        return 1

    def _swiglu(self, stream: int, gu, out, rows: int) -> int:
        """out = silu(gate) * up on the fused gate/up projection."""
        check(self.k_swiglu(stream, _ptr(gu), _ptr(out), rows, self.I), "lade_swiglu")
        return 1

    def _commit(self, stream: int, commit) -> int:
        """State update at the end of the step, by `commit`:
        False: none (the sampling path decides on the host);
        "sample": verification + residual draw on device (Philox), then the decision's commit and KV compaction;
        True on one GPU: fused verify + accept + update, then KV compaction;
        True under LP: the local verify, then the exchange and the replicated commit when NCCL runs in the library
        (otherwise generate() calls _lp_commit outside the step)."""
        lib = self.lib
        if not commit:
            return 0
        if commit == "sample" and self._cuts_on():
            w = _cabi.LadeWarpers(float(self.sample_temperature), int(self.sample_top_k), float(self.sample_top_p),
                                  float(self.sample_min_p), float(self.sample_epsilon), float(self.sample_eta))
            check(self.k_sample_verify_warped(self._ctx, stream, _ptr(self.logits), self.V, self.V, _ptr(self.am),
                                              _ptr(self.meta), C.byref(w), _ptr(self.rng_state), _ptr(self.dec_dev),
                                              _ptr(self.debug_uniforms), _ptr(self.debug_cuts)),
                  "lade_sample_verify_warped")
            check(lib.lade_commit_decision(self._ctx, stream, _ptr(self.dec_dev), _ptr(self.meta), _ptr(self.res)),
                  "lade_commit_decision")
            n = 2
        elif commit == "sample":
            check(self.k_sample_verify(self._ctx, stream, _ptr(self.logits), self.V, self.V, _ptr(self.am), _ptr(self.meta),
                                       float(self.sample_temperature), int(self.sample_top_k), float(self.sample_top_p),
                                       _ptr(self.rng_state), _ptr(self.dec_dev), _ptr(self.debug_uniforms)),
                  "lade_sample_verify")
            check(lib.lade_commit_decision(self._ctx, stream, _ptr(self.dec_dev), _ptr(self.meta), _ptr(self.res)),
                  "lade_commit_decision")
            n = 2
        elif self.DW == 1:
            check(lib.lade_accept_update(self._ctx, stream, _ptr(self.am), _ptr(self.meta), _ptr(self.res)),
                  "lade_accept_update")
            n = 1
        else:
            check(lib.lade_lp_verify(self._ctx, stream, _ptr(self.am), _ptr(self.meta), _ptr(self.lp_send)),
                  "lade_lp_verify")
            return 1 + (self._lp_commit(stream) if self._nccl_comm else 0)
        check(lib.lade_kv_compact(stream, _ptr(self.res), _ptr(self.kv[0, 0]), _ptr(self.kv[0, 1]),
                                  self.kv.stride(0), self.L, self.nkv, self.kv_capacity, self.D, max(self.GS - 1, 1)),
              "lade_kv_compact")
        return n + 1

    def _capture(self, stream: int, commit) -> int:
        """With capture on, copy the row each token the step emitted was decided from into capture_buf (after the
        commit has written res).  Off, or on a step the host decides (commit=False), nothing is launched."""
        if not (self.capture_on and commit):
            return 0
        buf = self.capture_buf
        check(self.k_capture_rows(self._ctx, stream, _ptr(self.logits), self.V, self.V, _ptr(self.ids),
                                  _ptr(self.lm_rows), _ptr(self.meta), _ptr(self.res), int(commit == "sample"),
                                  _ptr(buf), buf.stride(0), buf.shape[0]), "lade_capture_rows")
        return 1

    def _cuts_on(self) -> bool:
        """Any of MinP / epsilon / eta set: the sampling step runs lade_sample_verify_warped."""
        return bool(self.sample_min_p or self.sample_epsilon or self.sample_eta)

    def _lp_comm_create(self) -> None:
        """In-library NCCL communicator for the per-step record exchange (lade_lp_exchange): rank 0 draws the unique
        id, torch.distributed carries its 128 bytes to the other ranks (set-up only), every rank joins.  With
        LADE_LP_TORCH_ALLGATHER=1 (or no NCCL in the process) the exchange falls back to dist.all_gather_into_tensor."""
        import os as _os
        import torch.distributed as dist
        if _os.environ.get("LADE_LP_TORCH_ALLGATHER", "0") == "1" or not self.lib.lade_nccl_available():
            return
        if dist.get_backend(self.pg) != "nccl":          # gloo groups (CPU tests) have no device collectives
            return
        uid = torch.zeros(128, dtype=torch.uint8)
        if self.rank == 0:
            buf = (C.c_char * 128)()
            check(self.lib.lade_nccl_unique_id(buf), "lade_nccl_unique_id")
            uid = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        uid_dev = uid.to(self.dev)
        src = dist.get_global_rank(self.pg, 0) if self.pg is not None else 0
        dist.broadcast(uid_dev, src=src, group=self.pg)
        raw = bytes(uid_dev.cpu().numpy().tobytes())
        check(self.lib.lade_nccl_comm_create(raw, self.DW, self.rank, C.byref(self._nccl_comm)), "lade_nccl_comm_create")

    @property
    def lp_in_library(self) -> bool:
        return bool(self._nccl_comm)

    def _lp_commit(self, stream: int) -> int:
        """LP: one all-gather of the fixed-size per-rank records, then the replicated commit."""
        if self._nccl_comm:      # ncclAllGather on the compute stream, inside the library (graph-capturable)
            check(self.lib.lade_lp_exchange(self._ctx, stream, self._nccl_comm, _ptr(self.lp_send), _ptr(self.lp_recv)),
                  "lade_lp_exchange")
        else:
            import torch.distributed as dist
            dist.all_gather_into_tensor(self.lp_recv, self.lp_send, group=self.pg)
        check(self.lib.lade_lp_commit(self._ctx, stream, _ptr(self.lp_recv), _ptr(self.meta), _ptr(self.res)),
              "lade_lp_commit")
        return 1

    @staticmethod
    def _parse_result(r) -> StepRecord:
        n_emit = int(r[_cabi.R_N_EMIT])
        return StepRecord(n_emit=n_emit, max_hit=int(r[_cabi.R_MAX_HIT]),
                          hits=[int(x) for x in r[_cabi.R_HITS:_cabi.R_HITS + n_emit]],
                          n_guess=int(r[_cabi.R_N_GUESS]), kv_len=int(r[_cabi.R_KV_LEN]), done=bool(r[_cabi.R_DONE]))

    def _read_result(self) -> StepRecord:
        self._pinned_res.copy_(self.res, non_blocking=True)
        torch.cuda.current_stream(self.dev).synchronize()
        return self._parse_result(self._pinned_res.numpy())

    def _enqueue_result_copy(self, slot: int) -> None:
        """Stream-ordered D2H copy of the step record into pinned slot `slot`, marked by an event."""
        self._pinned_ring[slot].copy_(self.res, non_blocking=True)
        self._res_events[slot].record(torch.cuda.current_stream(self.dev))

    def _wait_result(self, slot: int) -> StepRecord:
        self._res_events[slot].synchronize()
        return self._parse_result(self._pinned_ring[slot].numpy())

    def _steady_graph(self, commit: bool = True):
        if self._graph is None:
            self._graph = {}
        key = (commit, float(self.sample_temperature), int(self.sample_top_k), float(self.sample_top_p),
               float(self.sample_min_p), float(self.sample_epsilon), float(self.sample_eta)) \
            if commit == "sample" else (commit, self.processors_on)
        if self.capture_on:       # the capture launch bakes the buffer in: one graph per buffer
            key = key + (("capture", self.capture_buf.data_ptr(), self.capture_buf.shape[0]),)
        if key in self._graph:
            self._graph_n = self._graph[key][1]
            return self._graph[key][0]
        rows = self.q_steady
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(side):
            with torch.cuda.graph(g, stream=side):
                n = self._launch_step(rows, torch.cuda.current_stream(self.dev).cuda_stream, commit=commit)
        torch.cuda.current_stream(self.dev).wait_stream(side)
        self._graph[key] = (g, n)
        self._graph_n = n
        return g

    @torch.no_grad()
    def run_forward_step(self, step: int, n_prompt: int, commit: bool = True) -> None:
        """One step's launches (eager for the prefill / window-fill steps, graph replay afterwards)."""
        stream = torch.cuda.current_stream(self.dev).cuda_stream
        if step <= self.N - 3 or not self.use_cuda_graph:
            rows = self.lib.lade_step_rows_bound(C.byref(self._lcfg), n_prompt, step)
            if rows < 0:
                raise LadeError("lade_step_rows_bound failed")
            if rows > self.rows_cap:
                raise LadeError(f"step {step} needs {rows} rows but the engine buffers hold {self.rows_cap}")
            self.launches += self._launch_step(rows, stream, commit=commit, prefill=(step == 0))
        else:
            self._steady_graph(commit).replay()
            self.launches += self._graph_n

    def begin(self, prompt, max_length: int, eos_token_ids, window0, processors: Optional[dict] = None,
              capture_logits: bool = False) -> None:
        """Reset the device state for a generate() call (lade_ctx_reset), write the logits-processor record and size
        the buffers.  `capture_logits`: every step also copies the rows its tokens were decided from into capture_buf,
        max_length - P + N - 1 rows (a step may emit up to N - 2 tokens past max_length)."""
        P = len(prompt)
        if capture_logits and self.DW != 1:
            raise LadeError("logits capture is not supported with lookahead parallelism (DIST_WORKERS > 1): the "
                            "accepted n-gram's rows live on one rank")
        self.capture_on = bool(capture_logits)
        if self.capture_on:
            rows = max_length - P + self.GS
            if self.capture_buf is None or self.capture_buf.shape[0] < rows:
                self.capture_buf = torch.empty(rows, self.V, dtype=self.dt, device=self.dev)
        rec = processors_record(processors) if processors else None
        self._ensure_ctx(eos_token_ids)
        stream = torch.cuda.current_stream(self.dev).cuda_stream
        if rec is not None:
            check(self.lib.lade_processors_upload(stream, C.byref(rec), _ptr(self.proc_dev)), "lade_processors_upload")
        self.processors_on = rec is not None
        prompt_np = np.asarray(prompt, dtype=np.int32)
        win_np = np.asarray(list(window0), dtype=np.int32)
        check(self.lib.lade_ctx_reset(self._ctx, stream, prompt_np.ctypes.data, P, win_np.ctypes.data, len(win_np),
                                      max_length), "lade_ctx_reset")
        torch.cuda.current_stream(self.dev).synchronize()   # host buffers were consumed
        self.launches += 2 + int(self.pool_from_prompt)
        rows0 = int(self.lib.lade_step_rows_bound(C.byref(self._lcfg), P, 0))
        if rows0 > self.rows_cap:
            self._graph = None
            self._alloc(rows0)

    def draw_window(self, prompt, rng=None, window0=None):
        """Initial lookahead window: W+N-3 draws of random.choice(prompt), exactly as lade/decoding.py:887-902
        (same python RNG consumption); under LP rank 0's draw is broadcast (:905-906)."""
        rnd = rng or random
        if window0 is None:
            window0 = [rnd.choice(prompt) for _ in range(self.WCAP)]
        if self.DW > 1:
            import torch.distributed as dist
            wt = torch.tensor(list(window0), dtype=torch.int32, device=self.dev)
            dist.broadcast(wt, src=dist.get_global_rank(self.pg, 0) if self.pg is not None else 0, group=self.pg)
            window0 = wt.cpu().tolist()
        return list(window0)

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def generate(self, prompt_ids: Sequence[int], max_new_tokens: int, eos_token_ids: Sequence[int] = (),
                 rng: Optional[random.Random] = None, window0: Optional[Sequence[int]] = None,
                 stop_fn=None, sampling: Optional[dict] = None, processors: Optional[dict] = None,
                 capture_logits: bool = False) -> List[int]:
        """Greedy lookahead decoding; returns prompt + generated ids (trimmed to P + max_new_tokens).
        `stop_fn(ids) -> bool`: host-evaluated stopping criteria beyond max-length / EOS, checked after every step
        like lade/decoding.py:1215 (disables the one-step-deep host pipelining).
        `sampling={"temperature": T, "top_k": k, "top_p": p, "seed": s}`: the sampling loop (jacobi_sample_multilevel, lade/decoding.py:137) with
        the verification on device (lade_sample_verify, Philox stream seeded by `s`): same host loop, same CUDA graph
        replay per step, the only difference is the commit kernels at the end of the step.  Optional further keys
        "min_p" ([0, 1]), "epsilon" and "eta" (0 or (0, 1)): HF's MinP / Epsilon / Eta warpers after top-p, 0 = off
        (lade_sample_verify_warped when any is on).
        `processors={"penalty": p, "prompt_ignore_length": k, "ngram_size": n, "min_length": m, "eos_token_id": [...]}`
        (every key optional): HF's greedy RepetitionPenalty / NoRepeatNGram / MinLength logits processors, applied on
        device to every row the step's verification reads, each against the prefix that row stands for
        (lade_argmax_processed).  "min_length" is the length below which the eos ids score -inf
        (max(min_length, prompt_length + min_new_tokens) for HF's two processors).  Greedy and one GPU only.
        `capture_logits=True`: afterwards `last_logits` is a [generated tokens, V] view (model dtype) whose row j is the
        lm-head row generated token j was decided from -- the model's next-token logits for exactly that token's
        prefix, since lookahead is lossless -- captured on device inside the step graph (lade_capture_rows); the next
        capturing generate() reuses the buffer.  One GPU only."""
        prompt = [int(t) for t in prompt_ids]
        P = len(prompt)
        max_length = P + int(max_new_tokens)
        if max_length > self.max_total_len:
            raise LadeError(f"prompt+max_new_tokens={max_length} exceeds engine capacity {self.max_total_len}")
        commit = True
        if processors and sampling is not None:
            raise LadeError("logits processors are supported on the greedy path only (not with sampling=)")
        if processors and self.DW != 1:
            raise LadeError("logits processors are not supported with lookahead parallelism (DIST_WORKERS > 1)")
        if sampling is not None:
            if self.DW != 1:
                raise LadeError("the sampling path has no lookahead parallelism (reference: replicas only)")
            T = float(sampling.get("temperature", 1.0))
            if not T > 0:
                raise LadeError("temperature must be > 0")
            top_k, top_p = int(sampling.get("top_k", 0) or 0), float(sampling.get("top_p", 1.0))
            if top_k < 0 or not 0.0 < top_p <= 1.0:
                raise LadeError("top_k must be >= 0 and top_p in (0, 1]")
            cuts = [float(sampling.get(k, 0.0) or 0.0) for k in ("min_p", "epsilon", "eta")]
            if not 0.0 <= cuts[0] <= 1.0:
                raise LadeError(f"min_p must be in [0, 1] (got {sampling.get('min_p')})")
            for name, v in zip(("epsilon", "eta"), cuts[1:]):
                if not (v == 0.0 or 0.0 < v < 1.0):
                    raise LadeError(f"{name} must be 0 (off) or in (0, 1) (got {v})")
            self.sample_temperature, self.sample_top_k, self.sample_top_p = T, top_k, top_p
            self.sample_min_p, self.sample_epsilon, self.sample_eta = cuts
            commit = "sample"
        self.last_logits = None
        self.begin(prompt, max_length, eos_token_ids, self.draw_window(prompt, rng, window0), processors,
                   capture_logits=capture_logits)
        if sampling is not None:
            self.rng_state.copy_(torch.tensor([int(sampling.get("seed", 0)) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64))
        stream = torch.cuda.current_stream(self.dev).cuda_stream
        out = list(prompt)
        self.last_records = []
        # The decode state lives on the device, so step i+1 never needs the host's view of step i: it is queued
        # while the host is still waiting for step i's record (the 48-int D2H copy), which hides the host
        # turn-around (~60 us per step).  Step i+1 is NOT queued when step i certainly ends the generation
        # (every step emits >= 1 token); if the end comes early (EOS, multi-token accept) the one surplus step runs
        # on a finished state, where the commit kernels are no-ops, and its record is dropped.
        inflight: List[int] = []      # result slots of queued steps, oldest first
        queued = 0                    # steps queued so far
        step = 0                      # steps whose record has been read
        guard = max_new_tokens + self.N + 4
        # lookahead parallelism: pipelined too when the exchange is in-library (every rank replays the same graph in the
        # same order: the decisions are replicated); the torch all-gather fallback keeps the synchronous loop
        pipelined = self.pipeline_host and (self.DW == 1 or bool(self._nccl_comm)) and stop_fn is None

        def enqueue():
            nonlocal queued
            self.run_forward_step(queued, P, commit=commit)
            if self.DW > 1 and not self._nccl_comm:       # torch all-gather fallback: outside the graph
                self.launches += self._lp_commit(stream)
            slot = queued & 1
            self._enqueue_result_copy(slot)
            inflight.append(slot)
            queued += 1

        enqueue()
        while True:
            certainly_last = (len(out) - P) + 1 >= max_new_tokens
            if pipelined and len(inflight) == 1 and not certainly_last:
                enqueue()
            rec = self._wait_result(inflight.pop(0))
            self.last_records.append(rec)
            out.extend(rec.hits)
            step += 1
            if rec.done or (stop_fn is not None and stop_fn(out[:max_length])):
                break
            if step > guard:
                raise LadeError("decode loop did not terminate (device state corrupt?)")
            if not inflight:
                enqueue()
        if inflight:                  # surplus speculative step: let it drain, ignore its record
            torch.cuda.current_stream(self.dev).synchronize()
            inflight.clear()
        self.last_steps = step
        if self.capture_on:
            self.last_logits = self.capture_buf[:len(out[:max_length]) - P]
        return out[:max_length]                                   # lade/decoding.py:1221-1225
