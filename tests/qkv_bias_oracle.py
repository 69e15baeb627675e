"""Qwen2 / Qwen2.5 restatements for the tests: the oracle's forward with q/k/v projection biases, the bias term of the
float64 projection bound, and the rounding points of lade_rope_append_bias.

* ``BiasOracle``: ``oracle.llama_ref.OracleLlama`` whose forward adds ``self_attn.{q,k,v}_proj.bias`` when the weights
  hold them (Qwen2Attention: ``nn.Linear(..., bias=True)`` on q, k and v, none on o_proj), the same way the oracle picks
  up Qwen3's q_norm.  Without biases in the weights it is OracleLlama itself, value for value.  With bf16 / fp16 weights
  the biased projection is ``F.linear(x, w, b)``, one rounding of the sum, HF's rounding point; with float64 weights it is
  a float64 forward.
* ``linear_fp64``: ``oracle.llama_ref.linear_fp64`` with an optional bias: ref = a . w^T + b, and the bound charges the
  one more fp32 addition (of the bias to the accumulator) on a partial sum of magnitude at most sum_k |a_k w_k| + |b|.
  Without a bias it returns exactly what ``oracle.llama_ref.linear_fp64`` returns.
* ``biased``: x = T(acc + float(b)) in fp32, the first step of lade_rope_append_bias; ``rope_bias``: then RoPE of q and
  k with every op rounded to T (tests/qknorm_restatement.rope), V as x.
"""
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import llama_ref as LR

QKV = ("q_proj", "k_proj", "v_proj")


def linear_fp64(a: torch.Tensor, w: torch.Tensor, dtype, bias: Optional[torch.Tensor] = None
                ) -> Tuple[torch.Tensor, torch.Tensor]:
    """(ref, bound) of nn.Linear in float64 for a kernel that accumulates in fp32, adds `bias` (model dtype) to the
    accumulator and rounds once to `dtype`.  See oracle.llama_ref.linear_fp64 for the bound without a bias."""
    ref, bound = LR.linear_fp64(a, w, dtype)
    if bias is None:
        return ref, bound
    bd = bias.double()
    ref = ref + bd
    mag = a.double().abs() @ w.double().abs().t() + bd.abs()
    bound = 0.5 * LR.ulp(ref, dtype) + (LR.linear_gamma(a.shape[-1]) + 2.0 ** -23) * mag
    return ref, bound


class BiasOracle(LR.OracleLlama):
    """OracleLlama with Qwen2's q/k/v projection biases (see the module docstring)."""

    def __init__(self, cfg, weights, device="cpu", rope_dtype=None):
        super().__init__(cfg, weights, device=device, rope_dtype=rope_dtype)
        self.qkv_bias = "model.layers.0.self_attn.q_proj.bias" in self.w

    def _qkv(self, i: int, x: torch.Tensor, q_len: int):
        p = f"model.layers.{i}.self_attn."
        out = []
        for name, heads in zip(QKV, (self.nh, self.nkv, self.nkv)):
            b = self.w.get(p + name + ".bias") if self.qkv_bias else None
            out.append(F.linear(x, self.w[p + name + ".weight"], b).view(q_len, heads, self.D).transpose(0, 1))
        return out


def biased(acc: torch.Tensor, bias: torch.Tensor, dtype) -> torch.Tensor:
    """T(acc + float(bias)): acc fp32 [..., C], bias [C] in `dtype`; the sum in fp32, one rounding."""
    return (acc.float() + bias.float()).to(dtype)


def rope_bias(acc: torch.Tensor, bias: torch.Tensor, nh: int, nkv: int, D: int, cos, sin, dtype):
    """(q [nh, rows, D], k [nkv, rows, D], v [nkv, rows, D]) of lade_rope_append_bias for the fp32 projection acc
    [rows, (nh + 2 nkv) D], with cos / sin [rows, D] in `dtype` (the rows' positions)."""
    from qknorm_restatement import rope
    rows = acc.shape[0]
    x = biased(acc, bias, dtype).view(rows, nh + 2 * nkv, D).transpose(0, 1)
    q, k, v = x[:nh], x[nh:nh + nkv], x[nh + nkv:]
    return rope(q, cos, sin), rope(k, cos, sin), v
