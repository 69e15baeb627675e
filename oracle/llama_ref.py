"""TEST INFRASTRUCTURE ONLY -- torch restatement of the floating-point side of lade's step.

Functional Llama forward over the lookahead step rows, following the reference's eager path
(``/root/reference/lade/models/modeling_llama.py``): RMSNorm ``:222-227``, rotary tables
``:240-266`` and application ``:342-346``, attention ``:492-558`` (QK^T, ``/ sqrt(d)`` as a
division ``:523``, additive ``finfo.min`` mask ``:536``, fp32 softmax cast back ``:539``, PV
``:541``), SwiGLU MLP ``:378``, decoder layer ``:858-889``, final norm + lm_head ``:1240,1541-1544``.

It is the checker for the CUDA kernels (same rounding points as the reference, so it is the "torch
reference" of the floating-point kernels) and, timed on the host cores, the ``cpu_baseline`` /
``--impl reference`` leg of ``bench.py``.  The product package never imports it.

Parity status: PINNED through ``tests/golden`` (per-step argmax tokens and final ids of the
unmodified reference model run from /root/reference with the same seeded weights).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from . import lookahead as LA


def init_weights(cfg: dict, seed: int = 0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Seeded random-init Llama weights (normal(0, 0.02), norms = 1), name-sorted draw order.

    Identical draws to ``oracle.ref_shim.build_reference_model`` so the unmodified reference model
    and this functional restatement share weights bit-for-bit.
    """
    H, L, I, V = cfg["hidden"], cfg["layers"], cfg["inter"], cfg["vocab"]
    nh, nkv = cfg["heads"], cfg.get("kv_heads") or cfg["heads"]
    D = cfg.get("head_dim") or H // nh
    shapes = {"lm_head.weight": (V, H), "model.embed_tokens.weight": (V, H), "model.norm.weight": (H,)}
    for i in range(L):
        p = f"model.layers.{i}."
        shapes[p + "input_layernorm.weight"] = (H,)
        shapes[p + "post_attention_layernorm.weight"] = (H,)
        shapes[p + "self_attn.q_proj.weight"] = (nh * D, H)
        shapes[p + "self_attn.k_proj.weight"] = (nkv * D, H)
        shapes[p + "self_attn.v_proj.weight"] = (nkv * D, H)
        shapes[p + "self_attn.o_proj.weight"] = (H, nh * D)
        shapes[p + "mlp.gate_proj.weight"] = (I, H)
        shapes[p + "mlp.up_proj.weight"] = (I, H)
        shapes[p + "mlp.down_proj.weight"] = (H, I)
    g = torch.Generator().manual_seed(seed)
    w = {}
    for name in sorted(shapes):
        shp = shapes[name]
        if len(shp) >= 2:
            w[name] = (torch.randn(shp, generator=g) * 0.02).to(dtype)
        else:
            w[name] = torch.ones(shp, dtype=dtype)
    return w


def rope_tables(D: int, max_pos: int, theta: float, dtype, device,
                table_dtype=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """cos/sin caches as modeling_llama.py:240-256 (fp32 math, then cast to the model dtype :264-265).

    `table_dtype` (default `dtype`) is the precision the tables are rounded to before they are widened to `dtype`: a
    float64 forward takes either the tables a 16-bit model uses (the device step's operands) or the fp32 ones that HF
    computes for a float64 model."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, D, 2).float() / D))
    t = torch.arange(max_pos, dtype=inv_freq.dtype)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    td = dtype if table_dtype is None else table_dtype
    return emb.cos().to(td).to(dtype).to(device), emb.sin().to(td).to(dtype).to(device)


def _acc_dtype(dtype):
    """Where the reference computes in fp32 (RMSNorm statistics, softmax): fp32, or float64 for a float64 forward."""
    return torch.float64 if dtype == torch.float64 else torch.float32


def rms_norm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    dt = x.dtype
    xf = x.to(_acc_dtype(dt))
    var = xf.pow(2).mean(-1, keepdim=True)
    xf = xf * torch.rsqrt(var + eps)
    return w * xf.to(dt)


def rotate_half(x):
    x1 = x[..., : x.shape[-1] // 2]
    x2 = x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def additive_mask(vis: torch.Tensor, kv_len: int, dtype) -> torch.Tensor:
    """[q, kv_len+q] additive mask: 0 where visible, finfo(dtype).min elsewhere (modeling :122,205-206)."""
    q = vis.shape[0]
    m = torch.full((q, q), torch.finfo(dtype).min, dtype=dtype, device=vis.device)
    m.masked_fill_(vis, 0)
    if kv_len > 0:
        m = torch.cat([torch.zeros(q, kv_len, dtype=dtype, device=vis.device), m], dim=-1)
    return m


# A float64 attention whose score block [H, q, kv] would exceed this many elements runs over groups of heads: the
# result is the same per head, and a 2900-row prefill at 32 heads stays within a few GB of temporaries.
F64_SCORE_CHUNK = 1 << 27


def eager_attention(q, k, v, mask, n_rep: int = 1):
    """Reference eager attention numerics on [H, q, D] x [Hkv, kv, D] (modeling_llama.py:520-541)."""
    H, R, T = q.shape[0], q.shape[1], k.shape[1]
    if q.dtype == torch.float64 and H * R * T > F64_SCORE_CHUNK and H > n_rep:
        hk = max(1, F64_SCORE_CHUNK // (n_rep * R * T)) * n_rep          # whole GQA groups per chunk
        return torch.cat([eager_attention(q[h:h + hk], k[h // n_rep:(h + hk) // n_rep],
                                          v[h // n_rep:(h + hk) // n_rep], mask, n_rep) for h in range(0, H, hk)])
    if n_rep > 1:
        k = k.repeat_interleave(n_rep, dim=0)
        v = v.repeat_interleave(n_rep, dim=0)
    D = q.shape[-1]
    s = torch.matmul(q, k.transpose(1, 2)) / math.sqrt(D)
    s = s + mask
    p = torch.nn.functional.softmax(s, dim=-1, dtype=_acc_dtype(q.dtype)).to(q.dtype)
    return torch.matmul(p, v)


# ---- float64 attention and its error bound ------------------------------------------------------------------------
# Constants of the bound (attention_fp64).  Derivation, per output element o[r, d] = sum_j p_j v_jd:
#   C_ULP = 1:  the final rounding to the model dtype costs <= 0.5 ulp; the other 0.5 ulp covers a result that lands
#               in the binade above o_ref (its ulp is twice as large) and the fp32 arithmetic of the normalisation.
#   C_SPREAD = 4:  every probability is rounded to the model dtype once (reference and kernels alike), a relative error
#               delta_j with |delta_j| <= u_T (absolute <= half the smallest subnormal step below the normal range).
#               Normalising by the sum of the rounded (impl 2) or unrounded (impl 1) probabilities, or rounding after
#               the normalisation (impl 3), turns them into sum_j delta_j p_j (v_jd - o_d) or sum_j delta_j p_j v_jd:
#               a sum of independent, zero-mean errors.  Round-to-nearest of a value with a spread mantissa has an RMS
#               relative error of about 0.42 u_T, so 4 * u_T * ||p (|v| + |o|)|| is a >= 9 sigma event; even Hoeffding's
#               inequality, which only uses |delta_j| <= u_T, puts it at <= 2 exp(-8) per element.
#   SCORE_WINDOW = 2^-20:  the kernels form T(T(raw) * fp32(1/sqrt(D))) with raw summed in fp32, the reference T(T(q.k) /
#               sqrt(D)).  A score within 2^-20 (relative) of a rounding midpoint of either rounding -- or, for the
#               first one, within the worst-case fp32 error D * 2^-24 * sum_i |q_i k_i| of the dot product -- may round
#               the other way; the bound adds what that other rounding does to the output, for those scores only:
#               p_j (e^Delta_j - 1)(|v_jd| + |o_d|) for a score moved by Delta_j.  That is the whole first-order effect
#               of the flip, so a flip that happens uses all of it: C_AMB = 2 keeps the margin the other terms have.
#   the floor:  2^-20 * sum_j p_j |v_jd| for the fp32 accumulation of P.V (<= 24 tile partial sums, each <= 2^-24
#               relative, plus the split merge), and 2^-100 so that a row that sees nothing (o = 0) divides cleanly.
C_ULP, C_SPREAD, C_AMB, SCORE_WINDOW = 1.0, 4.0, 2.0, 2.0 ** -20
_DT_INFO = {torch.bfloat16: (7, -126, 2.0 ** -8, 2.0 ** -134), torch.float16: (10, -14, 2.0 ** -11, 2.0 ** -25)}


def ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of the model dtype `dtype` at |x| (float64), subnormal range included."""
    mant, emin, _, _ = _DT_INFO[dtype]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** (emin - mant))))
    return torch.exp2(e.clamp_min(emin) - mant)


def _round_alternative(x: torch.Tensor, dtype, window: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(T(x), the other rounding of x where x lies within `window` of the midpoint between T(x) and its neighbour on
    x's side, else T(x)), both float64."""
    r = x.to(dtype)
    rd = r.double()
    toward = torch.sign(x - rd) * torch.where(rd < 0, -1.0, 1.0)          # +1: step the magnitude up
    bits = r.view(torch.int16).to(torch.int32) + toward.to(torch.int32)
    alt = bits.to(torch.int16).view(dtype).double()
    ambiguous = (toward != 0) & (rd != 0) & ((x - 0.5 * (rd + alt)).abs() <= window) & torch.isfinite(alt)
    return rd, torch.where(ambiguous, alt, rd)


def visibility(step_vis: torch.Tensor, kv_len: int, q_rows: Optional[int] = None) -> torch.Tensor:
    """[q_rows, kv_len + q_len] bool: every row sees the cache; the step block as given.  Rows past q_len (PAD rows of
    a fixed-shape step) see the cache and nothing of the step."""
    q_len = step_vis.shape[0]
    q_rows = q_len if q_rows is None else q_rows
    vis = torch.zeros(q_rows, kv_len + q_len, dtype=torch.bool, device=step_vis.device)
    vis[:, :kv_len] = True
    vis[:q_len, kv_len:] = step_vis
    return vis


def attention_fp64(q, k, v, vis, dtype) -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's attention (modeling_llama.py:520-541) in float64 with the reference's score rounding, and a
    per-element bound on how far an honest model-dtype kernel may be from it (constants above).

    q [Hq, R, D], k/v [Hkv, T, D] (model dtype values), vis [R, T] bool (or [Hq, R, T]).
    Returns (o_ref, bound), both float64 [Hq, R, D].  s = T(T(q.k) / sqrt(D)), masked scores are -inf, softmax and P.V
    in float64; a row that sees nothing gives 0."""
    _, _, u, eta = _DT_INFO[dtype]
    Hq, R, D = q.shape
    n_rep = Hq // k.shape[0]
    qd = q.double()
    kd = k.double().repeat_interleave(n_rep, dim=0)
    vd = v.double().repeat_interleave(n_rep, dim=0)
    vis = vis.to(q.device).expand(Hq, R, kd.shape[1])
    raw = qd @ kd.transpose(1, 2)
    w_raw = torch.maximum(SCORE_WINDOW * raw.abs(), D * 2.0 ** -24 * (qd.abs() @ kd.abs().transpose(1, 2)))
    r1, r1_alt = _round_alternative(raw, dtype, w_raw)
    s, s_alt = _round_alternative(r1 / math.sqrt(D), dtype, SCORE_WINDOW * (r1 / math.sqrt(D)).abs())
    s2, s2_alt = _round_alternative(r1_alt / math.sqrt(D), dtype, SCORE_WINDOW * (r1_alt / math.sqrt(D)).abs())
    delta = torch.maximum((s_alt - s).abs(), torch.maximum((s2 - s).abs(), (s2_alt - s).abs()))
    s = s.masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - torch.where(torch.isfinite(m), m, 0.0))
    l = e.sum(-1, keepdim=True)
    p = torch.where(l > 0, e / torch.where(l > 0, l, 1.0), 0.0)
    o = p @ vd
    va, oa = vd.abs(), o.abs()
    # per-probability rounding error: relative u, absolute eta (below the normal range), never more than p itself
    err_p = torch.minimum(p, torch.maximum(u * p, torch.full_like(p, eta)))
    err_p = torch.where(vis, err_p, 0.0)
    e2 = err_p * err_p
    spread = (e2 @ (vd * vd) + 2 * oa * (e2 @ va) + oa * oa * e2.sum(-1, keepdim=True)).clamp_min(0).sqrt()
    amb = torch.where(vis, p * torch.expm1(delta), 0.0)
    amb_term = amb @ va + oa * amb.sum(-1, keepdim=True)
    bound = C_ULP * ulp(o, dtype) + C_SPREAD * spread + C_AMB * amb_term + 2.0 ** -20 * (p @ va) + 2.0 ** -100
    return o, bound


def bound_ratio(got: torch.Tensor, o_ref: torch.Tensor, bound: torch.Tensor) -> torch.Tensor:
    """|got - o_ref| / bound, float64 (NaN or inf in `got` gives inf)."""
    err = (got.double() - o_ref).abs()
    return torch.where(torch.isfinite(err), err / bound, math.inf)


# Acceptance of a kernel output against attention_fp64: no element beyond its bound, and on average well inside it (an
# honest kernel sits near 0.1; a systematic error such as a 1 % scale moves the mean, not only the tail).
MAX_RATIO, MEAN_RATIO = 1.0, 0.25


def within_bound(got, o_ref, bound, mean_ratio: float = MEAN_RATIO) -> Tuple[bool, float, float]:
    """(passes, max ratio, mean ratio) of `got` against (o_ref, bound) of attention_fp64 or linear_fp64."""
    ratio = bound_ratio(got, o_ref, bound)
    mx, mean = ratio.max().item(), ratio.mean().item()
    return mx <= MAX_RATIO and mean <= mean_ratio, mx, mean


# ---- float64 projection GEMM and its error bound ------------------------------------------------------------------
# A correctly rounded output alone has a mean error of a quarter ulp, 0.5 of the bound's half-ulp term, so the mean
# criterion of a GEMM output is 0.55: where the accumulation term is small an honest kernel sits at 0.5, lower
# elsewhere; an output rounded any other way than to nearest does not.
LINEAR_MEAN_RATIO = 0.55


def linear_gamma(K: int) -> float:
    """Relative weight of sum_k |a_k w_k| in the bound of linear_fp64 (derivation there)."""
    return (K / 16 + 4 + 8) * 2.0 ** -23


def linear_fp64(a: torch.Tensor, w: torch.Tensor, dtype) -> Tuple[torch.Tensor, torch.Tensor]:
    """nn.Linear without bias in float64, c = a . w^T for a [M, K], w [N, K] (model dtype values), and a per-element
    bound on how far a kernel that accumulates in fp32 and rounds once to `dtype` may be from it.

    Returns (ref, bound), float64 [M, N]:
        bound = ulp_T(ref) / 2 + gamma * (|a| . |w|^T),    gamma = (K / 16 + 4 + 8) * 2^-23.
    * ulp_T(ref) / 2: the single rounding of the fp32 result to the model dtype.  (A result that the accumulation error
      d pushes over a power of two rounds with the coarser spacing, but the power of two itself is representable, so
      the rounding moves it by at most d more; the slack of gamma covers that.)
    * gamma: the products of two model-dtype values are exact in fp32.  Every k16 step of the tensor core adds one
      16-term sum to the accumulator: K / 16 sequential fp32 additions; the 16-term sum counts as a 4-level tree; up to
      8 split-K partials add at most 8 more.  Each addition is charged 2^-23, not the 2^-24 of round-to-nearest,
      because the tensor core may truncate where IEEE would round.  All of them act on partial sums of magnitude at
      most sum_k |a_k w_k|.
    Integer operands whose partial sums stay below 2^24 make every addition exact whatever the order: then a kernel
    must return T(ref) bit for bit, which the exact probes of the tests use."""
    ad, wd = a.double(), w.double()
    ref = ad @ wd.t()
    bound = 0.5 * ulp(ref, dtype) + linear_gamma(a.shape[-1]) * (ad.abs() @ wd.abs().t())
    return ref, bound


# ---- float64 RMSNorm and SwiGLU with the kernels' rounding points -------------------------------------------------
# Both return the result and, per element, the other admissible result: where the value that is rounded to the model
# dtype lies so close to a rounding midpoint that the fp32 arithmetic in front of it may tip it either way, the
# neighbouring model-dtype number is as correct as the nearest one.  A kernel output is right iff it equals the first
# tensor, or the second where the two differ; `unexplained` counts the rest.
NORM_WINDOW_ULPS, SILU_WINDOW_ULPS = 8, 8


def rms_norm_fp64(x, delta, w, eps: float, dtype):
    """LlamaRMSNorm with the fused residual add (modeling_llama.py:222-227, :883-889), T = `dtype`:
        h = T(x + delta)  (torch's model-dtype add; delta may be None), n = T(h * rstd), out = T(w * n),
        rstd = 1 / sqrt(mean(h^2) + fp32(eps)) in float64.
    Returns (h, out, out_alt).  n has an alternative where h * rstd is within a relative (hidden + 8) * 2^-24 of a
    rounding midpoint: the fp32 sum of `hidden` squares in any order is off by at most hidden * 2^-24 relative, and
    the division, the addition of eps, rsqrtf (2 ulp) and the final product add less than 8 * 2^-24.  w * n is the
    product of two model-dtype numbers, exact in fp32, so the last rounding has no alternative of its own."""
    h = x if delta is None else x + delta
    hd = h.double()
    hidden = h.shape[-1]
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    rstd = 1.0 / torch.sqrt(hd.pow(2).mean(-1, keepdim=True) + eps32)
    v = hd * rstd
    n, n_alt = _round_alternative(v, dtype, (hidden + NORM_WINDOW_ULPS) * 2.0 ** -24 * v.abs())
    wd = w.double()
    return h, (wd * n).to(dtype), (wd * n_alt).to(dtype)


_LOG_FLT_MAX = math.log(float(torch.finfo(torch.float32).max))


def swiglu_fp64(gate_up: torch.Tensor, dtype):
    """LlamaMLP's act_fn(gate) * up (modeling_llama.py:378) on the fused [rows, 2 * inter] projection, T = `dtype`:
        s = T(silu(g)), out = T(s * u),   silu(g) = g / (1 + exp(-g)) in float64.
    Returns (out, out_alt).  s has an alternative where silu(g) is within a relative 8 * 2^-24 of a rounding midpoint
    (expf 2 ulp, the addition, the division, with room to spare).  The reference evaluates silu in fp32, where exp(-g)
    overflows for g < -88.72 and the quotient is -0; the restatement says -0 there too (bf16 could represent the
    float64 value, about -1e-37).  s * u is exact in fp32; an fp16 product beyond 65504 is inf in both."""
    inter = gate_up.shape[-1] // 2
    g, u = gate_up[..., :inter].double(), gate_up[..., inter:].double()
    v = g / (1.0 + torch.exp(-g))
    v = torch.where(-g > _LOG_FLT_MAX, -torch.zeros_like(g), v)
    s, s_alt = _round_alternative(v, dtype, SILU_WINDOW_ULPS * 2.0 ** -24 * v.abs())
    return (s * u).to(dtype), (s_alt * u).to(dtype)


def unexplained(got: torch.Tensor, main: torch.Tensor, alt: torch.Tensor) -> Tuple[int, int]:
    """(elements of `got` that equal neither `main` nor `alt`, elements that needed `alt`); NaN equals only NaN."""
    def same(p, q):
        return (p == q) | (torch.isnan(p) & torch.isnan(q))
    is_main = same(got, main)
    is_alt = same(got, alt)
    return int((~is_main & ~is_alt).sum()), int((~is_main & is_alt).sum())


class OracleLlama:
    """Functional Llama with a growing KV cache, driven by ``oracle.lookahead.greedy_lookahead``.

    Qwen3 too: `cfg["head_dim"]` when heads * head_dim != hidden, and the per-head q/k RMSNorm in front of RoPE
    (Qwen3Attention) when the weights hold ``self_attn.q_norm.weight`` / ``k_norm.weight``.

    bf16 / fp16 weights give the reference's rounding points.  float64 weights give a float64 forward with no fp32
    step inside (RMSNorm statistics, softmax and logits stay float64); it needs `rope_dtype`, the precision of its
    RoPE tables: the model dtype of the 16-bit model it stands for (the device step's tables), or torch.float32
    (HF's tables for a float64 model).  The embedding and lm_head of a float64 forward may stay in the model dtype:
    the forward widens only the embedding rows it gathers, and lm_head one vocabulary chunk at a time, so a checkpoint
    vocabulary of 152064 costs no float64 copy of either."""

    LM_CHUNK = 16384            # vocabulary rows of lm_head widened at a time

    def __init__(self, cfg: dict, weights: Dict[str, torch.Tensor], device="cpu", rope_dtype=None):
        self.cfg = cfg
        self.dev = torch.device(device)
        self.w = {k: v.to(self.dev) for k, v in weights.items()}
        self.dtype = self.w["model.norm.weight"].dtype
        if self.dtype == torch.float64 and rope_dtype is None:
            raise ValueError("a float64 OracleLlama needs rope_dtype (the model dtype's tables or torch.float32)")
        self.H, self.L = cfg["hidden"], cfg["layers"]
        self.nh = cfg["heads"]
        self.nkv = cfg.get("kv_heads") or cfg["heads"]
        self.D = cfg.get("head_dim") or self.H // self.nh
        self.eps = cfg.get("eps", 1e-5)
        self.qk_norm = "model.layers.0.self_attn.q_norm.weight" in self.w
        self.cos, self.sin = rope_tables(self.D, cfg.get("max_pos", 4096), cfg.get("rope_theta", 10000.0),
                                         self.dtype, self.dev, table_dtype=rope_dtype)
        self.reset()

    def reset(self):
        self.k_cache: List[Optional[torch.Tensor]] = [None] * self.L
        self.v_cache: List[Optional[torch.Tensor]] = [None] * self.L
        self.last_hidden = None
        self.last_attn_io = None

    def _qkv(self, i: int, x: torch.Tensor, q_len: int):
        """q [nh, q_len, D], k and v [nkv, q_len, D] of layer i (the hook a model with projection biases overrides)."""
        p = f"model.layers.{i}.self_attn."
        return [torch.nn.functional.linear(x, self.w[p + name + "_proj.weight"]).view(q_len, heads, self.D).transpose(0, 1)
                for name, heads in (("q", self.nh), ("k", self.nkv), ("v", self.nkv))]

    def _lm_head(self, h: torch.Tensor) -> torch.Tensor:
        lm = self.w["lm_head.weight"]
        if lm.dtype == h.dtype:
            return torch.nn.functional.linear(h, lm)
        out = torch.empty(h.shape[0], lm.shape[0], dtype=h.dtype, device=h.device)
        for c in range(0, lm.shape[0], self.LM_CHUNK):
            out[:, c:c + self.LM_CHUNK] = h @ lm[c:c + self.LM_CHUNK].to(h.dtype).t()
        return out

    # -- one forward over the step rows, returns fp32 logits [q, V] (float64 for a float64 model) ---
    def forward_rows(self, ids, pos, vis_mask: torch.Tensor, kv_len: int, capture_layer: int = -1,
                     logit_rows: Optional[List[int]] = None):
        """`logit_rows`: the step rows whose logits are returned (in that order), default all of them."""
        w, dt = self.w, self.dtype
        ids_t = torch.as_tensor(ids, dtype=torch.long, device=self.dev)
        pos_t = torch.as_tensor(pos, dtype=torch.long, device=self.dev)
        q_len = ids_t.numel()
        h = w["model.embed_tokens.weight"][ids_t].to(dt)
        mask = additive_mask(vis_mask.to(self.dev), kv_len, dt)
        cos, sin = self.cos[pos_t], self.sin[pos_t]
        for i in range(self.L):
            p = f"model.layers.{i}."
            res = h
            x = rms_norm(h, w[p + "input_layernorm.weight"], self.eps)
            q, k, v = self._qkv(i, x, q_len)
            if self.qk_norm:                    # Qwen3RMSNorm over each head, before the rotary embedding
                q = rms_norm(q, w[p + "self_attn.q_norm.weight"], self.eps)
                k = rms_norm(k, w[p + "self_attn.k_norm.weight"], self.eps)
            q = (q * cos) + (rotate_half(q) * sin)
            k = (k * cos) + (rotate_half(k) * sin)
            if self.k_cache[i] is not None and kv_len > 0:
                k = torch.cat([self.k_cache[i][:, :kv_len], k], dim=1)
                v = torch.cat([self.v_cache[i][:, :kv_len], v], dim=1)
            self.k_cache[i], self.v_cache[i] = k, v
            o = eager_attention(q, k, v, mask, self.nh // self.nkv)
            if i == capture_layer:
                self.last_attn_io = (q.clone(), k.clone(), v.clone(), o.clone())
            o = o.transpose(0, 1).reshape(q_len, self.nh * self.D)
            h = res + torch.nn.functional.linear(o, w[p + "self_attn.o_proj.weight"])
            res = h
            x = rms_norm(h, w[p + "post_attention_layernorm.weight"], self.eps)
            g = torch.nn.functional.linear(x, w[p + "mlp.gate_proj.weight"])
            u = torch.nn.functional.linear(x, w[p + "mlp.up_proj.weight"])
            h = res + torch.nn.functional.linear(torch.nn.functional.silu(g) * u, w[p + "mlp.down_proj.weight"])
        h = rms_norm(h, w["model.norm.weight"], self.eps)
        self.last_hidden = h
        if logit_rows is not None:
            h = h[torch.as_tensor(logit_rows, dtype=torch.long, device=self.dev)]
        logits = self._lm_head(h)
        return logits if dt == torch.float64 else logits.float()

    # -- StepFn / CompactFn for oracle.lookahead.greedy_lookahead ---------------------------------
    def step_fn(self, lay: LA.StepLayout, kv_len: int):
        vis = torch.from_numpy(LA.step_mask(lay))
        logits = self.forward_rows(lay.ids, lay.pos, vis, kv_len)
        self.last_logits = logits
        q = lay.q_len
        lg = lay.n_guess_tok
        window = lay.level_sizes[-1]
        out_tok = int(torch.argmax(logits[lay.n_input - 1]))
        inp = torch.argmax(logits[q - lg - window:q - lg], dim=-1).tolist()
        guess = torch.argmax(logits[q - lg:], dim=-1).tolist() if lg > 0 else []
        return out_tok, inp, guess

    def compact_fn(self, dst: int, src: int, n: int, new_len: int):
        for i in range(self.L):
            if n > 0:
                self.k_cache[i][:, dst:dst + n] = self.k_cache[i][:, src:src + n].clone()
                self.v_cache[i][:, dst:dst + n] = self.v_cache[i][:, src:src + n].clone()
            self.k_cache[i] = self.k_cache[i][:, :new_len]
            self.v_cache[i] = self.v_cache[i][:, :new_len]

    # -- plain autoregressive greedy (comparator; SURVEY.md App. C) --------------------------------
    def plain_greedy(self, prompt, max_new: int):
        self.reset()
        ids = list(prompt)
        kv = 0
        feed = ids
        for _ in range(max_new):
            n = len(feed)
            vis = torch.tril(torch.ones(n, n, dtype=torch.bool))
            logits = self.forward_rows(feed, list(range(kv, kv + n)), vis, kv)
            kv += n
            nxt = int(torch.argmax(logits[-1]))
            ids.append(nxt)
            feed = [nxt]
        return ids
